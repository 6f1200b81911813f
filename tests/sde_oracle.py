"""Oracles of SDE-DPM-Solver++ (`DPM_Solver(..., algorithm_type="sde-dpmsolver++")`) -- TEST INFRASTRUCTURE.

* `SdeOracle`: the numpy executor (every model type and guidance form) with the SDE update of dpm_step_sde. The model
  stage is the parent executor's (its buffered value, rounded to the state dtype); the update is the LIN1 / DIFF2 / MS3
  expression of include/dpm_solver_b200.h plus cz*z in fp32, each op rounded. z is drawn by the contract, at the launch:
  `torch.empty_like(x, dtype=torch.float32).normal_(generator=g)` on x's device. On the GPU box that is the draw the
  kernel replays in registers, so the executor checks each launch bit for bit; on the CPU it is the CPU generator's.
  `draws` keeps every z it drew, so a float64 run can be fed the same values. The update's output is laid out as the
  CUDA backend lays it out (channels_last when x is, and no preallocated output says otherwise), so that the next
  update's draw follows the same storage order.
* `kdiff_sde`: k-diffusion's `sample_dpmpp_2m_sde` / `sample_dpmpp_3m_sde` loops restated in float64 in the VE
  coordinates x^ = x/alpha, sigma^ = sigma/alpha (t = -log sigma^ = lambda), with the first update(s) of lower order
  and the noise z_i given.
"""
import dataclasses
import math

import numpy as np
import torch

from dpm_solver_b200._lib import FORM_DIFF2, FORM_LIN1, FORM_MS3, FORM_NONE
from fdg_oracle import FDGOracle
from oracle_backend import _np

f32 = np.float32


class SdeOracle(FDGOracle):
    """The numpy executor with dpm_step_sde."""

    def __init__(self):
        super().__init__()
        self.draws = []

    def draw(self, a):
        """The noise of launch `a`: the contract's draw from its generator."""
        return torch.empty_like(a.x, dtype=torch.float32).normal_(generator=a.sde.generator)

    def step(self, a):
        if getattr(a, "sde", None) is None:
            return super().step(a)
        if a.form not in (FORM_LIN1, FORM_DIFF2, FORM_MS3) or a.c0_on_old:
            raise ValueError("an SDE step is a multistep LIN1 / DIFF2 / MS3 update")
        ref = a.reference_tensor()
        sdt = a.state_dtype or a.x.dtype
        if a.n_model > 0:
            b = dataclasses.replace(a, sde=None, form=FORM_NONE, want_m_out=True, out=None, out2=None)
            m_out = super().step(b)[0]
            T0 = _np(m_out)
        else:
            self.launches += 1
            self.log.append((a.form, 0))
            m_out, T0 = None, _np(a.m0)
        z = self.draw(a)
        self.draws.append(z.detach().cpu().clone())
        x, m1, m2, zz = _np(a.x), _np(a.m1), _np(a.m2), _np(z)
        A, c0, c1, c2 = f32(a.a), f32(a.c0), f32(a.c1), f32(a.c2)
        w0, w1, w2, w3 = f32(a.w0), f32(a.w1), f32(a.w2), f32(a.w3)
        if a.form == FORM_LIN1:
            o = A * x + c0 * T0
        elif a.form == FORM_DIFF2:
            o = (A * x + c0 * T0) + c1 * (w0 * (T0 - m1))
        else:
            D10 = w0 * (T0 - m1)
            D11 = w1 * (m1 - m2)
            dd = D10 - D11
            o = ((A * x + c0 * T0) + c1 * (D10 + w2 * dd)) + c2 * (w3 * dd)
        o = o + f32(a.sde.cz) * zz
        out = torch.from_numpy(np.ascontiguousarray(o.astype(f32))).to(sdt).reshape(ref.shape).to(ref.device)
        if _launch_layout(a) == "cl":
            # the state the launch writes keeps its layout, and the next update's draw follows that storage order
            out = out.contiguous(memory_format=torch.channels_last if out.dim() == 4 else torch.channels_last_3d)
        if a.out is not None:
            a.out.copy_(out.reshape(a.out.shape))
            out = a.out
        if a.out2 is not None:
            a.out2.copy_(out.reshape(a.out2.shape))
        if m_out is not None:
            m_out = m_out.to(ref.device) if a.want_m_out else None
        return m_out, out


def _launch_layout(a):
    """The storage order of a launch's outputs, as the CUDA backend picks it: x's dense layout ("c" or "cl"), or
    row-major when x has none or a preallocated output is laid out otherwise."""
    from dpm_solver_b200.ops import CudaBackend
    layout = CudaBackend._layout(a.reference_tensor()) or "c"
    for t in (a.out, a.m_out, a.out2):
        if t is not None and CudaBackend._layout(t) != layout:
            layout = "c"
    return layout


def kdiff_sde(x_T, denoise, alphas, sigmas, zs, eta, order, solver_type="dpmsolver"):
    """float64 k-diffusion DPM++ 2M / 3M SDE (order 2 / 3; order 1 is its first update alone) over the grid of
    marginals alphas[i], sigmas[i] (i = 0..N), in x-space at both ends. denoise(x, i) -> x0 (float64 numpy, x-space at
    grid point i); zs[i] the noise of update i + 1. Returns the x of every grid point."""
    al = [float(a) for a in alphas]
    sg = [float(s) for s in sigmas]
    sh = [s / a for s, a in zip(sg, al)]                   # sigma^
    lam = [-math.log(s) for s in sh]
    xh = np.asarray(x_T, dtype=np.float64) / al[0]
    out = [xh * al[0]]
    d1 = d2 = None
    h1 = h2 = None
    for i in range(len(al) - 1):
        den = denoise(xh * al[i], i)
        h = lam[i + 1] - lam[i]
        h_eta = h * (eta + 1)
        x_new = math.exp(-h_eta) * xh + (-math.expm1(-h_eta)) * den      # (sigma^_t/sigma^_s)*exp(-eta*h)*x + ...
        if order >= 3 and h2 is not None:
            r0, r1 = h1 / h, h2 / h
            d1_0 = (den - d1) / r0
            d1_1 = (d1 - d2) / r1
            D1 = d1_0 + (d1_0 - d1_1) * r0 / (r0 + r1)
            D2 = (d1_0 - d1_1) / (r0 + r1)
            phi_2 = math.expm1(-h_eta) / h_eta + 1
            phi_3 = phi_2 / h_eta - 0.5
            x_new = x_new + phi_2 * D1 - phi_3 * D2
        elif order >= 2 and h1 is not None:
            r = h1 / h
            d = (den - d1) / r
            if order >= 3 or solver_type == "taylor":            # heun (and 3M's order-2 warm-up)
                x_new = x_new + (math.expm1(-h_eta) / h_eta + 1) * d
            else:                                                # midpoint
                x_new = x_new + 0.5 * (-math.expm1(-h_eta)) * d
        if eta:
            x_new = x_new + np.asarray(zs[i], dtype=np.float64) * sh[i + 1] * math.sqrt(-math.expm1(-2 * h * eta))
        xh = x_new
        d2, d1 = d1, den
        h2, h1 = h1, h
        out.append(xh * al[i + 1])
    return out
