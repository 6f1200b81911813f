"""Oracles of the EDM path (`NoiseScheduleEDM`, `model_type="edm"`) -- TEST INFRASTRUCTURE.

* `EDMOracle`: the numpy executor with every guidance form and dpm_step_unipc (unipc_oracle.UniPCOracle, itself the
  flow executor) plus DPM_PARAM_EDM as include/dpm_solver_b200.h states it: value = alpha_e*xe + sigma_e*out, each op
  rounded, in either space (the words say which), each output converted before the combine, a rescaled combine
  converted after it, no eps -> x0 division.
* `reference_solver`: the UNMODIFIED reference DPM_Solver (updates, time grids, order schedules, thresholding, adaptive
  loop) on a subclass of its NoiseScheduleVP whose marginal methods are NoiseScheduleEDM's closed forms, driven by a
  test-side model function that converts each network output with the two words in eager torch ops and combines the
  converted values; a three-line subclass returns that x0 instead of dividing (:439). `karras_steps` gives it the
  product's skip_type="karras" grid, restated from its docstring.
"""
import copy
import math

import numpy as np
import torch

from flow_oracle import FlowOracle
from oracle import ref_loader
from test_cfg_rescale import ratio64
from unipc_oracle import UniPCOracle

f32 = np.float32
PARAM_FLOW, PARAM_EDM = 4, 5


class EDMOracle(UniPCOracle):
    _edm = False

    def _flow(self, a, out, xe):
        if not self._edm:
            return FlowOracle._flow(a, out, xe)
        with np.errstate(all="ignore"):
            return (f32(a.alpha_e) * xe + f32(a.sigma_e) * out).astype(f32)

    def _model_value(self, a, thr=None):
        if a.param != PARAM_EDM:
            return super()._model_value(a, thr)
        # the flow executor's guidance forms, with the EDM conversion in place of the flow one
        b = copy.copy(a)
        b.param = PARAM_FLOW
        self._edm = True
        try:
            return super()._model_value(b, thr)
        finally:
            self._edm = False


# ---- the reference on the EDM schedule ---------------------------------------------------------------------------------

def reference_schedule(sigma_min=0.002, sigma_max=80., sigma_data=0.5, rho=7., total_N=1000):
    """The reference's NoiseScheduleVP with NoiseScheduleEDM's closed forms (its docstring's op order) in place of its
    marginal methods."""
    ref = ref_loader.load("dpm_solver_pytorch")
    c = float(np.float32(1. / total_N))
    smin_r = sigma_min ** (1. / rho)
    span_r = sigma_max ** (1. / rho) - smin_r
    sd2 = sigma_data * sigma_data

    class RefEDM(ref.NoiseScheduleVP):
        def __init__(self):
            super().__init__("linear")
            self.schedule, self.total_N, self.T = "edm", total_N, 1.
            self.sigma_data = sigma_data

        def sigma(self, t):
            u = (t - c) / (1. - c)
            return (smin_r + u * span_r) ** rho

        def _r(self, t):
            s = self.sigma(t)
            return torch.sqrt(s * s + sd2)

        def marginal_alpha(self, t):
            return 1. / self._r(t)

        def marginal_std(self, t):
            return self.sigma(t) / self._r(t)

        def marginal_log_mean_coeff(self, t):
            return -torch.log(self._r(t))

        def marginal_lambda(self, t):
            return -torch.log(self.sigma(t))

        def inverse_lambda(self, lamb):
            s = torch.exp(-lamb)
            u = (s ** (1. / rho) - smin_r) / span_r
            return u * (1. - c) + c

    ns = RefEDM()
    ns.input_time = lambda t: 0.25 * torch.log(ns.sigma(t))
    return ns


def words(ns, t, x0_space):
    """The per-sample conversion words at labels t: fp32 marginals, each word formed in double and rounded once."""
    al, sg, sd = ns.marginal_alpha(t).double(), ns.marginal_std(t).double(), ns.sigma_data
    if x0_space:
        return (sd * sd * al).float(), (sd * sg).float()
    return sg.float(), (-sd * al).float()


def expand(v, x):
    return v.reshape((-1,) + (1,) * (x.dim() - 1))


def reference_model(net, ns, x0_space, guidance=None, calls=None, phi=0.0):
    """model_fn(x, t_continuous) -> the solver-space value, in eager fp32 torch.
    guidance: None (the network takes (x, t)), or dict(uc=, conds=[c1..cK], scales=float | [B] list | [s1..sK] list,
    kind="scalar" | "per_sample" | "multi"); the network then takes (x, t, c)."""
    def conv(v, x, t):
        a, b = words(ns, t, x0_space)
        return expand(a, x) * x + expand(b, x) * v

    def fn(x, t):
        t_in = ns.input_time(t)
        if guidance is None:
            if calls is not None:
                calls.append((tuple(x.shape), t_in.tolist()))
            return conv(net(x, t_in), x, t)
        n = len(guidance["conds"]) + 1
        x_in, tt = torch.cat([x] * n), torch.cat([t_in] * n)
        if calls is not None:
            calls.append((tuple(x_in.shape), tt.tolist()))
        outs = net(x_in, tt, torch.cat([guidance["uc"], *guidance["conds"]])).chunk(n)
        kind, s = guidance["kind"], guidance["scales"]
        if kind == "multi":
            tu = conv(outs[0], x, t)
            T = tu
            for sk, o in zip(s, outs[1:]):
                T = T + float(np.float32(sk)) * (conv(o, x, t) - tu)
            return T
        u, cc = outs
        if kind == "scalar" and phi:
            g = u + s * (cc - u)
            r = torch.from_numpy(ratio64(cc.numpy(), g.numpy())).reshape(-1, *([1] * (g.dim() - 1)))
            return conv(phi * (g * r) + (1.0 - phi) * g, x, t)
        tc, tu = conv(cc, x, t), conv(u, x, t)
        if kind == "scalar":
            return tu + s * (tc - tu)
        sv = expand(torch.tensor(s, dtype=torch.float32), x)
        return torch.where(sv == 1, tc, tu + sv * (tc - tu))      # a scale of 1: the conditional output alone
    return fn


def karras_steps(ns, t_T, t_0, N):
    """skip_type="karras" as the product's get_time_steps documents it."""
    lT = ns.marginal_lambda(torch.tensor(t_T)).item()
    l0 = ns.marginal_lambda(torch.tensor(t_0)).item()
    r = torch.linspace(math.exp(-lT / 7.), math.exp(-l0 / 7.), N + 1).pow(7.)
    return ns.inverse_lambda(-torch.log(r))


def reference_solver(net, ns, algorithm_type, thresholding=False, **model_kw):
    """The reference DPM_Solver on the EDM schedule. Its noise model is the eps-space function; the data prediction
    (dpmsolver++, denoise_to_zero) takes the x0-space function as it is instead of dividing (:439)."""
    ref = ref_loader.load("dpm_solver_pytorch")
    x0_fn = reference_model(net, ns, True, **model_kw)

    class EDMSolver(ref.DPM_Solver):
        def data_prediction_fn(self, x, t):
            x0 = x0_fn(x, t.expand((x.shape[0])))
            return x0 if self.correcting_x0_fn is None else self.correcting_x0_fn(x0, t)

        def get_time_steps(self, skip_type, t_T, t_0, N, device):
            if skip_type == "karras":
                return karras_steps(self.noise_schedule, t_T, t_0, N).to(device)
            return super().get_time_steps(skip_type, t_T, t_0, N, device)

    # (dpmsolver++ never calls the eps-space function; handing it no `calls` keeps the log to the calls that happen)
    eps_kw = dict(model_kw) if algorithm_type == "dpmsolver" else dict(model_kw, calls=None)
    return EDMSolver(reference_model(net, ns, False, **eps_kw), ns, algorithm_type=algorithm_type,
                     correcting_x0_fn="dynamic_thresholding" if thresholding else None)
