"""UniPC multistep sampling (Zhao et al., "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling of
Diffusion Models", NeurIPS 2023, arXiv:2302.04867) on the fused sm_90a step path.

    fn = model_wrapper(unet, ns, guidance_type="classifier-free", condition=c, unconditional_condition=uc,
                       guidance_scale=7.5)
    x0 = UniPC(fn, ns, algorithm_type="dpmsolver++", variant="bh2").sample(x_T, steps=10, order=2)

The method
----------
The grid t_0 = t_T > t_1 > ... > t_N is `get_time_steps`' (DPM_Solver's). alpha_i, sigma_i, lambda_i are the fp32
values of `plan.Marginals` (the update formulas take exp(log alpha), the conversion alpha_t, as in DPM_Solver).
m_i is the converted model value at (x~_i, t_i) -- x0 for "dpmsolver++", eps for "dpmsolver" -- with the
parameterisation, classifier-free guidance, dynamic thresholding and flow conversion of DPM_Solver's fused step.

Step i runs from t_{i-1} to t_i with order p_i = min(order, i), capped at N + 1 - i when `lower_order_final` is set.
This is not DPM_Solver's multistep rule, which lowers the final orders only when steps < 10: UniPC lowers them for
every number of steps. Its scalars:

    h = lambda_i - lambda_{i-1};  hh = -h (data prediction) or +h (noise prediction);  h_phi_1 = expm1(hh)
    B = hh ("bh1") or expm1(hh) ("bh2")
    r_k = (lambda_{i-1-k} - lambda_{i-1}) / h for k = 1 .. p-1, r_p = 1
    h_phi_k = h_phi_1/hh - 1;  f = 1
    for j in 1..p:  R_j = (r_1^(j-1), ..., r_p^(j-1));  b_j = h_phi_k*f/B;  f = f*(j+1);  h_phi_k = h_phi_k/hh - 1/f
    predictor weights rho_p: [] (p = 1), [0.5] (p = 2), solve(R[:2, :2], b[:2]) (p = 3)
    corrector weights rho_c: [0.5] (p = 1), solve(R, b) (p >= 2)

With D_k = (m_{i-1-k} - m_{i-1}) / r_k and the base x_{i-1} (the corrected state; x_T at i = 1):

    predictor  x~_i = sigma_i/sigma_{i-1} x_{i-1} - alpha_i h_phi_1 m_{i-1} - alpha_i B sum_k rho_p_k D_k
    corrector  x_i  = sigma_i/sigma_{i-1} x_{i-1} - alpha_i h_phi_1 m_{i-1}
                      - alpha_i B (sum_{k<p} rho_c_k D_k + rho_c_p (m_i - m_{i-1}))          (i < N, after m_i)

(noise prediction: alpha_i/alpha_{i-1} and sigma_i in place of sigma_i/sigma_{i-1} and alpha_i). Without the corrector
x_i = x~_i. Step N is predictor only: there is no evaluation at t_N, and x~_N is the result. Step 1's predictor is
DPM-Solver's first update (plan._first, the fused LIN1 launch); UniP-2 with "bh2" and no corrector is
DPM-Solver(++)(2M) in exact arithmetic.

How it runs
-----------
Predictor and corrector share their base terms, so

    x_i = x~_i - alpha_i B (sum_{k<p} (rho_c_k - rho_p_k) D_k + rho_c_p (m_i - m_{i-1}))

and one launch per evaluation i = 1 .. N-1 (dpm_step_unipc) reads x~_i, the network output(s) and the buffers,
converts, corrects, rounds x_i to the state dtype in registers, and writes m_i and the next network input x~_{i+1}:
evaluation 0, one LIN1 launch, then N - 1 UniPC launches (plus the quantile launch per evaluation with dynamic
thresholding). The host folds every word of a launch -- signs, -alpha_i B (rho_c_k - rho_p_k)/r_k, the next
predictor's weights -- in fp64 from the fp32 marginals (a series where the h_phi recursion cancels) and rounds each
once to fp32; the kernel forms the buffer differences first, then the sums left to right, each op rounded.

Hooks: with `correcting_xt_fn` the launch runs the corrector only and writes x_i, the hook sees x_i, and a pure
predictor launch reads the hooked state. A custom `correcting_x0_fn` sees the materialised m_i (conversion launch,
hook, then the UniPC launch on the hooked value). `return_intermediate` returns x_T, the corrected x_1 .. x_{N-1}
and x_N.

Adaptive projected guidance (model_wrapper's apg_eta) runs with a scalar scale: per evaluation the words pass, one
launch that writes the buffered value m_i, then the UniPC launch reading it (n_model == 0). With dynamic thresholding
the guided x0 is materialised in fp32 first, then thresholded, then buffered.

CFG-Zero* (model_wrapper's cfg_zero_star) runs with a scalar scale: per evaluation the s* pass, one launch that
materialises the guided raw output g in fp32, then the UniPC launch converting g as a single network output at its own
state. Zero-init evaluations (cfg_zero_init_steps) are one-output launches on a raw output of 0, counted as in
DPM_Solver.

TCFG (model_wrapper's tcfg) runs with a scalar scale, as CFG-Zero* does: per evaluation the words pass (2 launches),
one launch that materialises the guided raw output g = us + w*(c - us), us = wu*u + wc*c, in fp32, then the UniPC
launch converting g as a single network output at its own state.

Frequency-decoupled guidance (model_wrapper's fdg_scales), shared or per-sample [B, N] scales: per evaluation the
pyramid pass (1 launch) gives g in the network's dtype, then the UniPC launch converts g as a single network output.

Not available (ValueError before any launch): per-sample guidance scales, several conditions, guidance masks,
guidance rescale, reference_rounding, plan_broadcast, orders outside 1..3, steps < order.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from . import plan as P
from .solver import DPM_Solver

__all__ = ["UniPC"]


@dataclass
class _Launch:
    """The words of one UniPC launch with the operands dpm_step_desc has no field for."""
    words: P.UniCoeffs
    m3: Optional[torch.Tensor] = None
    out_c: Optional[torch.Tensor] = None
    dev = None          # (scalars never live in device memory here)


class UniPC(DPM_Solver):
    _apg_materialise = True     # APG: the buffered value (+1 launch), then this launch on it; CFG-Zero*, TCFG: g (+1)

    def __init__(self, model_fn, noise_schedule, algorithm_type="dpmsolver++", variant="bh2", correcting_x0_fn=None,
                 correcting_xt_fn=None, thresholding_max_val=1., dynamic_thresholding_ratio=0.995, state_dtype=None):
        """UniPC multistep sampler. `algorithm_type` as in DPM_Solver ("dpmsolver++": data prediction,
        "dpmsolver": noise prediction); `variant` "bh1" (B(h) = h) or "bh2" (B(h) = expm1(h)); the other arguments
        as in DPM_Solver."""
        if variant not in ("bh1", "bh2"):
            raise ValueError("variant must be 'bh1' or 'bh2', got {!r}".format(variant))
        if algorithm_type == "sde-dpmsolver++":
            raise ValueError("UniPC has no SDE variant: algorithm_type='sde-dpmsolver++' is a DPM_Solver sampler")
        super().__init__(model_fn, noise_schedule, algorithm_type=algorithm_type, correcting_x0_fn=correcting_x0_fn,
                         correcting_xt_fn=correcting_xt_fn, thresholding_max_val=thresholding_max_val,
                         dynamic_thresholding_ratio=dynamic_thresholding_ratio, state_dtype=state_dtype)
        self.variant = variant

    @staticmethod
    def _fill_update(a, co, x, m1, m2) -> None:
        if not isinstance(co, _Launch):
            return DPM_Solver._fill_update(a, co, x, m1, m2)
        a.form, a.x, a.m1, a.m2 = co.words.form, x, m1, m2
        a.unipc, a.m3, a.out_c = co.words, co.m3, co.out_c

    def _check_supported(self, steps, order):
        if order not in (1, 2, 3):
            raise ValueError("UniPC order must be 1, 2 or 3, got {}".format(order))
        if steps < order:
            raise ValueError("UniPC needs steps >= order, got steps={} and order={}".format(steps, order))
        if self.reference_rounding:
            raise ValueError("reference_rounding=True is not available with UniPC")
        if self.plan_broadcast:
            raise ValueError("plan_broadcast=True is not available with UniPC")
        self._refuse("unipc")

    def inverse(self, x, steps=20, t_start=None, t_end=None, order=2, skip_type='time_uniform', lower_order_final=True,
                denoise_to_zero=False, use_corrector=True, return_intermediate=False):
        """Invert `x` from t_start (default 1/N) to t_end (default T): sample() over the reversed time range."""
        t_0 = 1. / self.noise_schedule.total_N if t_start is None else t_start
        t_T = self.noise_schedule.T if t_end is None else t_end
        assert t_0 > 0 and t_T > 0, "Time range needs to be greater than 0. For discrete-time DPMs, it needs to be in [1 / N, 1], where N is the length of betas array"
        return self.sample(x, steps=steps, t_start=t_0, t_end=t_T, order=order, skip_type=skip_type,
                           lower_order_final=lower_order_final, denoise_to_zero=denoise_to_zero,
                           use_corrector=use_corrector, return_intermediate=return_intermediate)

    def sample(self, x, steps=20, t_start=None, t_end=None, order=2, skip_type='time_uniform', lower_order_final=True,
               denoise_to_zero=False, use_corrector=True, return_intermediate=False):
        """Integrate the diffusion ODE from t_start (default T) to t_end (default 1/N) with UniPC multistep."""
        t_0 = 1. / self.noise_schedule.total_N if t_end is None else t_end
        t_T = self.noise_schedule.T if t_start is None else t_start
        assert t_0 > 0 and t_T > 0, "Time range needs to be greater than 0. For discrete-time DPMs, it needs to be in [1 / N, 1], where N is the length of betas array"
        self._check_supported(steps, order)
        self._check_fdg(x)
        ns, device, hook = self.noise_schedule, x.device, self.correcting_xt_fn
        intermediates = []
        self._xin_pair = None
        self._rr_run = 0
        self._prep_on = False           # UniPC launches are never frozen as prepared launches
        with torch.no_grad(), self._apg_scope():
            x = self._state(x)
            sd = x.dtype
            key = ("unipc", self.variant, steps, order, skip_type, t_T, t_0, lower_order_final, bool(use_corrector))

            def build():
                ts = self.get_time_steps(skip_type=skip_type, t_T=t_T, t_0=t_0, N=steps, device='cpu')
                marg = P.Marginals(ns, ts)
                orders = P.unipc_orders(steps, order, lower_order_final)
                first, launches = P.unipc_plan(self.algorithm_type, self.variant, marg, orders, bool(use_corrector))
                return ts, first, launches, list(zip(marg.alpha_e.tolist(), marg.sigma.tolist()))

            ts, first, launches, alsig = self._host_plan(key, build)
            _, _, ts_dev, _, tin = self._device_tables(key, ts, x.shape[0], device)
            tin = tin if tin is not None else [None] * (steps + 1)
            # evaluation 0 and step 1's predictor: DPM-Solver's first update, one fused LIN1 launch
            raw = self._evaluate(x, ts_dev[0], tin[0])
            xe = x
            if hook is not None:
                x = self._state_like(hook(x, ts_dev[0], 0), sd)
            if return_intermediate:
                intermediates.append(x)
            m, xt = self._post_model(raw, xe, ts_dev[0], alsig[0], first, x, want_m=steps > 1, dup_out=steps > 1)
            older = [m]                     # m_{i-1}, m_{i-2}, m_{i-3}: newest last
            for i in range(1, steps):
                raw = self._evaluate(xt, ts_dev[i], tin[i])
                w = launches[i - 1]
                m1 = older[-1]
                m2 = older[-2] if len(older) >= 2 else None
                m3 = older[-3] if len(older) >= 3 else None
                if hook is None:
                    # corrector of step i and predictor of step i+1: one launch
                    out_c = torch.empty_like(xt) if return_intermediate else None
                    m, x_next = self._post_model(raw, xt, ts_dev[i], alsig[i], _Launch(w, m3, out_c), xt, m1, m2,
                                                 want_m=i < steps - 1, dup_out=True)
                    xc = out_c
                else:
                    if w.pc > 0:
                        out_c = torch.empty_like(xt)
                        m, _ = self._post_model(raw, xt, ts_dev[i], alsig[i], _Launch(w.corrector_only(), m3, out_c),
                                                xt, m1, m2, want_m=True)
                    else:
                        m, _ = self._post_model(raw, xt, ts_dev[i], alsig[i])
                        out_c = xt
                    xc = self._state_like(hook(out_c, ts_dev[i], i), sd)
                    x_next = self._pure_update(_Launch(w.predictor_only()), xc, m, m1, m2)
                if return_intermediate:
                    intermediates.append(xc)
                older.append(m)
                if len(older) > 3:
                    older.pop(0)
                xt = x_next
            x = xt
            step = steps
            if hook is not None:
                x = self._state_like(hook(x, ts_dev[steps], steps), sd)
            if return_intermediate:
                intermediates.append(x)
            if denoise_to_zero:
                t, tin0, als0 = self._denoise_tables(t_0, x.shape[0], device)
                xs = self._state(x)
                x = self._post_model(self._evaluate(xs, t, tin0), xs, t, als0, x0=True)[0]
                if hook is not None:
                    x = hook(x, t, step + 1)
                if return_intermediate:
                    intermediates.append(x)
        self._net_input = None
        if return_intermediate:
            return x, intermediates
        return x
