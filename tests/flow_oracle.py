"""Oracles of the flow-matching path (`NoiseScheduleFlow`, `model_type="flow"`) -- TEST INFRASTRUCTURE.

* `FlowOracle`: the numpy executor with every guidance form (gpu_configs.FullOracle) plus DPM_PARAM_FLOW as
  include/dpm_solver_b200.h states it: x0 = xe - sigma_e*out (predict_x0) or eps = xe + alpha_e*out, each op rounded,
  each output converted before the combine, a rescaled combine converted after it, no eps -> x0 division.
* `reference_solver`: the UNMODIFIED reference DPM_Solver (updates, time grids, order schedules, thresholding, adaptive
  loop) on a subclass of its NoiseScheduleVP whose marginal methods are NoiseScheduleFlow's closed forms, driven by a
  test-side model function that converts each network output with the two torch ops above and combines the converted
  values; a three-line subclass returns that x0 instead of dividing (:439).
"""
import dataclasses

import numpy as np
import torch

from gpu_configs import FullOracle
from oracle import ref_loader
from oracle_backend import _np
from test_cfg_rescale import ratio64

f32 = np.float32
PARAM_FLOW = 4


class FlowOracle(FullOracle):
    @staticmethod
    def _flow(a, out, xe):
        with np.errstate(all="ignore"):
            if a.predict_x0:
                return (xe - f32(a.sigma_e) * out).astype(f32)
            return (xe + f32(a.alpha_e) * out).astype(f32)

    def _flow_one(self, a, xe, c, u, scale, ratio):
        """One scale (None: a single output) on numpy blocks; ratio: the rescale ratio per sample or None."""
        with np.errstate(all="ignore"):
            if u is None:
                return self._flow(a, c, xe)
            if ratio is not None:
                g = (u + f32(scale) * (c - u)).astype(f32)
                r = np.repeat(ratio, a.per_sample).reshape(g.shape)
                return self._flow(a, (f32(a.phi) * (g * r) + f32(1.0 - a.phi) * g).astype(f32), xe)
            tc, tu = self._flow(a, c, xe), self._flow(a, u, xe)
            return (tu + f32(scale) * (tc - tu)).astype(f32)

    def _model_value(self, a, thr=None):
        if a.param != PARAM_FLOW:
            return super()._model_value(a, thr)
        xe = _np(a.xe if a.xe is not None else a.x)
        c, u = _np(a.e_cond), _np(a.e_uncond) if a.n_model == 2 else None
        with np.errstate(all="ignore"):
            if a.e_conds is not None:
                tu = self._flow(a, u, xe)
                T = tu
                for s, e in zip(a.scales, a.e_conds):
                    T = (T + f32(s) * (self._flow(a, _np(e), xe) - tu)).astype(f32)
            elif a.guidance_b is not None:
                gb, rows = _np(a.guidance_b), []
                for b in range(gb.size):
                    one = gb[b] == 1            # the bypass: the converted conditional output alone
                    rows.append(self._flow_one(a, xe[b:b + 1], c[b:b + 1], None if one else u[b:b + 1], gb[b],
                                               None if a.ratio is None else _np(a.ratio)[b:b + 1]))
                T = np.concatenate(rows)
            else:
                T = self._flow_one(a, xe, c, u, a.guidance, None if a.ratio is None else _np(a.ratio))
            if a.predict_x0 and thr is not None:
                s = np.repeat(thr.reshape(-1), a.per_sample).reshape(T.shape)
                T = np.minimum(np.maximum(T, -s), s) / s
        return T.astype(f32)


# ---- the reference on the flow schedule ------------------------------------------------------------------------------

def reference_schedule(shift, time_scale=1000.0, total_N=1000):
    """The reference's NoiseScheduleVP with NoiseScheduleFlow's closed forms in place of its marginal methods."""
    ref = ref_loader.load("dpm_solver_pytorch")

    class RefFlow(ref.NoiseScheduleVP):
        def __init__(self):
            super().__init__("linear")
            self.schedule, self.total_N, self.T = "flow", total_N, 1. - 1. / total_N

        def marginal_std(self, t):
            return (shift * t) / (1. + (shift - 1.) * t)

        def marginal_alpha(self, t):
            return 1. - self.marginal_std(t)

        def marginal_log_mean_coeff(self, t):
            return torch.log(self.marginal_alpha(t))

        def marginal_lambda(self, t):
            return self.marginal_log_mean_coeff(t) - torch.log(self.marginal_std(t))

        def inverse_lambda(self, lamb):
            sigma = 1. / (1. + torch.exp(lamb))
            return sigma / (shift - (shift - 1.) * sigma)

    ns = RefFlow()
    ns.input_time = lambda t: time_scale * ns.marginal_std(t)
    return ns


def expand(v, x):
    return v.reshape((-1,) + (1,) * (x.dim() - 1))


def reference_model(net, ns, x0_space, guidance=None, calls=None, phi=0.0):
    """model_fn(x, t_continuous) -> the solver-space value, in eager fp32 torch.
    guidance: None (the network takes (x, t)), or dict(uc=, conds=[c1..cK], scales=float | [B] list | [s1..sK] list,
    kind="scalar" | "per_sample" | "multi"); the network then takes (x, t, c)."""
    def conv(v, x, t):
        if x0_space:
            return x - expand(ns.marginal_std(t), x) * v
        return x + expand(ns.marginal_alpha(t), x) * v

    def fn(x, t):
        B, t_in = x.shape[0], ns.input_time(t)
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
        u, c = outs
        if kind == "scalar" and phi:
            g = u + s * (c - u)
            r = torch.from_numpy(ratio64(c.numpy(), g.numpy())).reshape(-1, *([1] * (g.dim() - 1)))
            return conv(phi * (g * r) + (1.0 - phi) * g, x, t)
        tc, tu = conv(c, x, t), conv(u, x, t)
        if kind == "scalar":
            return tu + s * (tc - tu)
        sv = expand(torch.tensor(s, dtype=torch.float32), x)
        return torch.where(sv == 1, tc, tu + sv * (tc - tu))      # a scale of 1: the conditional output alone
    return fn


def reference_solver(net, ns, algorithm_type, thresholding=False, **model_kw):
    """The reference DPM_Solver on the flow schedule. Its noise model is the eps-space function; the data prediction
    (dpmsolver++, denoise_to_zero) takes the x0-space function as it is instead of dividing (:439)."""
    ref = ref_loader.load("dpm_solver_pytorch")
    x0_fn = reference_model(net, ns, True, **model_kw)

    class FlowSolver(ref.DPM_Solver):
        def data_prediction_fn(self, x, t):
            x0 = x0_fn(x, t.expand((x.shape[0])))
            return x0 if self.correcting_x0_fn is None else self.correcting_x0_fn(x0, t)

    # (dpmsolver++ never calls the eps-space function; handing it no `calls` keeps the log to the calls that happen)
    eps_kw = dict(model_kw) if algorithm_type == "dpmsolver" else dict(model_kw, calls=None)
    return FlowSolver(reference_model(net, ns, False, **eps_kw), ns, algorithm_type=algorithm_type,
                      correcting_x0_fn="dynamic_thresholding" if thresholding else None)
