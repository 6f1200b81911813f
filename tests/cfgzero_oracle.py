"""Oracles of CFG-Zero* (model_wrapper's cfg_zero_star) -- TEST INFRASTRUCTURE.

* `s_star_fsum`: the optimised scale of each sample from exactly rounded sums (math.fsum), the division in fp64 and
  one rounding to fp32: the formula of Fan, Zheng, Yeh and Liu, "CFG-Zero*: Improved Classifier-Free Guidance for Flow
  Matching Models" (2025, arXiv:2503.18886), with diffusers' 1e-8 in the denominator.
* `s_star_exact`: the same scale as dpm_cfgzero_scale sums it, operation for operation: words.cu's chunks, thread
  ownership, warp butterflies, warp order and chunk merge (apg_oracle.apg_sums_exact), so that it is bit-exact with
  the device.
* `cfgzero_combine`: g = us + w*(c - us), us = u*s*, in torch fp32 ops in that order (a per-sample scale of 1: c).
* `CFGZeroOracle`: the numpy executor (apg_oracle.APGOracle: every parameterisation, guidance form, dpm_step_unipc and
  APG) plus dpm_cfgzero_scale and dpm_step_cfgzero as include/dpm_solver_b200.h states them.
* `guided_net`: a network for the UNMODIFIED reference's guidance_type="uncond" wrapper that runs the real network
  on the doubled batch and returns the CFG-Zero* output, or 0 for its first K calls (zero-init).
"""
import copy
import math

import numpy as np
import torch

from apg_oracle import APGOracle, apg_sums_exact
from oracle_backend import _np

f32 = np.float32
EPS = 1e-8


def _storage_rows(v, ref=None):
    """[B, per_sample] fp32 rows of `v` in the order the device reads them: a channels_last tensor (laid out like
    `ref`, default v itself) holds each sample as (h, w, c)."""
    ref = v if ref is None else ref
    a = _np(v)
    if ref.dim() in (4, 5) and not ref.is_contiguous() and ref.is_contiguous(
            memory_format=torch.channels_last if ref.dim() == 4 else torch.channels_last_3d):
        a = a.transpose((0,) + tuple(range(2, ref.dim())) + (1,))
    return np.ascontiguousarray(a).reshape(a.shape[0], -1)


def s_star_fsum(c, u):
    """fp32 [B]: fl32(fsum(c*u) / (fsum(u*u) + 1e-8)) per sample, every product exact in fp64."""
    c, u = np.asarray(c, f32).reshape(len(c), -1), np.asarray(u, f32).reshape(len(u), -1)
    out = []
    for cb, ub in zip(c.astype(np.float64), u.astype(np.float64)):
        out.append(f32(math.fsum(cb * ub) / (math.fsum(ub * ub) + EPS)))
    return np.array(out, f32)


def s_star_exact(c, u):
    """fp32 [B] as the CFG-Zero* words pass (PairPass<2>) + k_cfgzero_final compute it, from [B, per_sample] rows
    in storage order."""
    uu, uc, _ = apg_sums_exact(np.asarray(u, f32), np.asarray(c, f32))   # (the fp64 product c*u == u*c, exactly)
    with np.errstate(all="ignore"):
        return (uc / (uu + EPS)).astype(f32)


def cfgzero_combine(out_c, out_u, s, w):
    """g in torch fp32, the contract's order; `s` fp32 [B]; `w` a python float or an fp32 [B] tensor (a row with
    w == 1 gets out_c alone)."""
    shape = (-1,) + (1,) * (out_c.dim() - 1)
    us = out_u * s.reshape(shape)
    if torch.is_tensor(w):
        wv = w.reshape(shape)
        return torch.where(wv == 1, out_c, us + wv * (out_c - us))
    return us + w * (out_c - us)


class CFGZeroOracle(APGOracle):
    """The numpy executor with dpm_cfgzero_scale (in the device's summation order, so its words are bit-exact) and
    dpm_step_cfgzero."""

    def cfgzero_scale(self, e_cond, e_uncond):
        self.launches += 2
        self.log.append(("cfgzero_scale", 2))
        return torch.from_numpy(s_star_exact(_storage_rows(e_cond), _storage_rows(e_uncond, e_cond)))

    def _model_value(self, a, thr=None):
        if getattr(a, "cfgzero_s", None) is None:
            return super()._model_value(a, thr)
        c, u, s = _np(a.e_cond), _np(a.e_uncond), _np(a.cfgzero_s)
        B = c.shape[0]
        shape = (B,) + (1,) * (c.ndim - 1)
        w = _np(a.guidance_b).reshape(shape) if a.guidance_b is not None else f32(a.guidance)
        with np.errstate(all="ignore"):
            us = (u * s.reshape(shape)).astype(f32)
            g = (us + (w * (c - us)).astype(f32)).astype(f32)
            g = np.where(w == 1, c, g)      # a sample whose scale is 1, per-sample or desc->guidance, gets c
        # the guided raw output is then converted like a single network output
        b = copy.copy(a)
        b.n_model, b.e_cond, b.e_uncond = 1, torch.from_numpy(np.ascontiguousarray(g)), None
        b.guidance_b = b.cfgzero_s = None
        b.guidance = 1.0
        return super()._model_value(b, thr)


def guided_net(net, uc, c, w, zero_steps=0, calls=None):
    """net_g(x, t_input) for a guidance_type="uncond" wrapper: the CFG-Zero* output of `net` on cat([x, x]) with
    cat([uc, c]) (s* in the device's exact order), or zeros for its first `zero_steps` calls. `calls`, when a list,
    receives one entry per real network call."""
    state = {"n": 0}

    def fn(x, t):
        state["n"] += 1
        if state["n"] <= zero_steps:
            return torch.zeros_like(x)
        if calls is not None:
            calls.append(tuple(x.shape))
        out_u, out_c = net(torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c])).chunk(2)
        s = torch.from_numpy(s_star_exact(_storage_rows(out_c), _storage_rows(out_u)))
        return cfgzero_combine(out_c, out_u, s, w)
    return fn
