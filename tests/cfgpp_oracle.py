"""Oracles of CFG++ (model_wrapper's cfg_pp) -- TEST INFRASTRUCTURE.

* `CFGPPOracle`: the numpy executor (cfgzero_oracle.CFGZeroOracle: every parameterisation, guidance form,
  dpm_step_unipc, APG and CFG-Zero*) plus dpm_step_cfgpp as include/dpm_solver_b200.h states it: U the x0 of e_uncond
  alone and G the guided x0, each from the executor's own single-output and CFG paths, rounded to the state type, then
  the update in its op order.
* `cfgpp_fp64`: an independent fp64 transcription of the paper's recurrences in VE coordinates (x^ = x/alpha,
  lambda = -log(sigma/alpha)) for a network given as x0 predictions.
"""
import copy
import math

import numpy as np
import torch

from cfgzero_oracle import CFGZeroOracle
from oracle_backend import _np, _round
from dpm_solver_b200._lib import FORM_DIFF2, FORM_LIN1

f32 = np.float32


class CFGPPOracle(CFGZeroOracle):
    """The numpy executor with dpm_step_cfgpp."""

    def step(self, a):
        if getattr(a, "cfgpp_g", None) is None:
            return super().step(a)
        assert a.form in (FORM_LIN1, FORM_DIFF2) and not a.c0_on_old and a.n_model == 2 and a.predict_x0
        assert a.thr is None and not a.raw_round and a.coef_dev is None
        self.launches += 1
        self.log.append(("cfgpp", a.form))
        ref = a.reference_tensor()
        sdt = a.state_dtype
        # U: the single-output step on e_uncond; G: the CFG step with the scalar (always combined) or per-sample scales
        u = copy.copy(a)
        u.n_model, u.e_cond, u.e_uncond, u.guidance_b, u.guidance, u.cfgpp_g = 1, a.e_uncond, None, None, 1.0, None
        g = copy.copy(a)
        g.cfgpp_g = None
        with np.errstate(all="ignore"):
            U = _round(self._model_value(u), sdt)
            G = _round(self._model_value(g), sdt)
            x = _np(a.x)
            A, c0, c1, w0, gw = f32(a.a), f32(a.c0), f32(a.c1), f32(a.w0), f32(a.cfgpp_g)
            o = (A * x + c0 * U) + gw * (G - U)
            if a.form == FORM_DIFF2:
                o = o + c1 * (w0 * (G - _np(a.m1)))
        m_out = torch.from_numpy(np.ascontiguousarray(U)).to(sdt).reshape(ref.shape) if a.want_m_out else None
        out = torch.from_numpy(np.ascontiguousarray(o.astype(f32))).to(sdt).reshape(ref.shape)
        if a.out is not None:
            a.out.copy_(out.reshape(a.out.shape))
            out = a.out
        if a.out2 is not None:
            a.out2.copy_(out.reshape(a.out2.shape))
        return m_out, out


def cfgpp_fp64(x0_pair, lam, alpha, x_T, order, solver_type="dpmsolver", lower_order_final=True):
    """The CFG++ multistep run in fp64 and VE coordinates. x0_pair(x, i) -> (G, U), the guided and the unconditional x0
    at grid point i (numpy, fp64); lam, alpha: the grid's lambda and alpha. Order 1 is the paper's DDIM CFG++
    x^' = G + e^-h*(x^ - U); order 2 adds -expm1(-h)/(2r)*(G - U_prev) ("dpmsolver") or
    (expm1(-h)/h + 1)/r*(G - U_prev) ("taylor")."""
    steps = len(lam) - 1
    x = np.asarray(x_T, np.float64)
    U_prev = None
    for i in range(steps):
        o = 1 if i == 0 or order == 1 else 2
        if order == 2 and lower_order_final and steps < 10 and i == steps - 1:
            o = 1
        G, U = x0_pair(x, i)
        h = lam[i + 1] - lam[i]
        xh = x / alpha[i]
        xn = G + math.exp(-h) * (xh - U)
        if o == 2:
            r = (lam[i] - lam[i - 1]) / h
            if solver_type == "dpmsolver":
                xn = xn - math.expm1(-h) / (2 * r) * (G - U_prev)
            else:
                xn = xn + (math.expm1(-h) / h + 1) / r * (G - U_prev)
        x = alpha[i + 1] * xn
        U_prev = U
    return x
