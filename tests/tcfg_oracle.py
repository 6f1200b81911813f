"""Oracles of TCFG (model_wrapper's tcfg) -- TEST INFRASTRUCTURE.

* `tcfg_svd_reference`: diffusers' `normalized_guidance` of TangentialClassifierFreeGuidance transcribed in float64
  with torch.linalg.svd: stack [c, u] per sample, zero the second right singular vector, project u on what is left.
  Returns the guided raw output g and the damped u'.
* `words_closed_form`: the closed form of the contract on given fp64 sums (A, B, C) = (||u||^2, <u, c>, ||c||^2),
  fp64 with each op rounded, each word rounded to fp32 once.
* `words_fsum`: the closed form on exactly rounded sums (math.fsum).
* `words_exact`: the words as dpm_tcfg_words computes them, operation for operation: words.cu's chunks,
  thread ownership, warp butterflies, warp order and chunk merge (apg_oracle.apg_sums_exact), then the closed form.
* `tcfg_combine`: g = us + w*(c - us), us = u*wu + c*wc, in torch fp32 ops in that order (a per-sample scale of 1: c).
* `TCFGOracle`: the numpy executor (cfgzero_oracle.CFGZeroOracle) plus dpm_tcfg_words and dpm_step_tcfg as
  include/dpm_solver_b200.h states them.
* `guided_net`: a network for the UNMODIFIED reference's guidance_type="uncond" wrapper that runs the real network on
  the doubled batch and returns the TCFG output, its words from `words_exact`.
"""
import copy
import math

import numpy as np
import torch

from apg_oracle import apg_sums_exact
from cfgzero_oracle import CFGZeroOracle, _storage_rows
from oracle_backend import _np

f32 = np.float32
NAN32 = np.array([0x7fffffff], np.uint32).view(np.float32)[0]    # the NaN k_tcfg_final writes


def tcfg_svd_reference(c, u, w):
    """(g, u') in float64 from diffusers' normalized_guidance: v = stack([c, u]) per sample, flattened; Vh of its SVD
    with row 1 zeroed; u' = (u_flat @ Vh^T) @ Vh; g = u' + w*(c - u'). `w`: a number or one value per sample."""
    c = torch.as_tensor(np.asarray(c, np.float64))
    u = torch.as_tensor(np.asarray(u, np.float64))
    B = c.shape[0]
    cf, uf = c.reshape(B, -1), u.reshape(B, -1)
    m = torch.stack([cf, uf], dim=1)                                # [B, 2, D]
    _, _, vh = torch.linalg.svd(m, full_matrices=False)             # [B, 2, D]
    vh = vh.clone()
    vh[:, 1] = 0
    up = ((uf.unsqueeze(1) @ vh.transpose(-2, -1)) @ vh).squeeze(1).reshape(u.shape)
    wv = torch.as_tensor(np.asarray(w, np.float64)).reshape((-1,) + (1,) * (c.dim() - 1))
    return (up + wv * (c - up)).numpy(), up.numpy()


def words_closed_form(A, B, C):
    """fp32 [n, 2] (wu, wc) from fp64 sums, as k_tcfg_final evaluates them."""
    A, B, C = (np.atleast_1d(np.asarray(v, np.float64)) for v in (A, B, C))
    out = np.empty((len(A), 2), f32)
    with np.errstate(all="ignore"):
        for i, (a, b, c) in enumerate(zip(A, B, C)):
            if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
                out[i] = NAN32
                continue
            h = 0.5 * (a - c)
            r = math.sqrt(h * h + b * b)
            if c >= a:
                p, q = b, (-h) + r
            else:
                p, q = h + r, b
            pp = p * p
            n2 = pp + q * q
            out[i] = (1.0, 0.0) if n2 == 0.0 else (f32(pp / n2), f32((p * q) / n2))
    return out


def words_fsum(c, u):
    """The closed form on exactly rounded sums of [B, per_sample] fp32 rows."""
    c = np.asarray(c, f32).reshape(len(c), -1).astype(np.float64)
    u = np.asarray(u, f32).reshape(len(u), -1).astype(np.float64)
    sums = [(math.fsum(ub * ub), math.fsum(ub * cb), math.fsum(cb * cb)) for cb, ub in zip(c, u)]
    return words_closed_form(*zip(*sums))


def words_exact(c, u):
    """fp32 [B, 2] as the TCFG words pass (PairPass<3>) + k_tcfg_final compute them, from [B, per_sample] rows in
    storage order. apg_sums_exact(R, c) sums R*R, R*c, c*c in the device's order: with R = u these are A, B, C."""
    A, B, C = apg_sums_exact(np.asarray(u, f32), np.asarray(c, f32))
    return words_closed_form(A, B, C)


def tcfg_combine(out_c, out_u, words, w):
    """g in torch fp32, the contract's order; `words` fp32 [B, 2]; `w` a python float or an fp32 [B] tensor (a row
    with w == 1 gets out_c alone)."""
    shape = (-1,) + (1,) * (out_c.dim() - 1)
    words = torch.as_tensor(words)
    wu, wc = words[:, 0].reshape(shape), words[:, 1].reshape(shape)
    us = out_u * wu + out_c * wc
    if torch.is_tensor(w):
        wv = w.reshape(shape)
        return torch.where(wv == 1, out_c, us + wv * (out_c - us))
    return us + w * (out_c - us)


class TCFGOracle(CFGZeroOracle):
    """The numpy executor with dpm_tcfg_words (in the device's summation order, so its words are bit-exact) and
    dpm_step_tcfg."""

    def tcfg_words(self, e_cond, e_uncond):
        self.launches += 2
        self.log.append(("tcfg_words", 2))
        return torch.from_numpy(words_exact(_storage_rows(e_cond), _storage_rows(e_uncond, e_cond)))

    def _model_value(self, a, thr=None):
        if getattr(a, "tcfg_w", None) is None:
            return super()._model_value(a, thr)
        c, u, tw = _np(a.e_cond), _np(a.e_uncond), _np(a.tcfg_w)
        B = c.shape[0]
        shape = (B,) + (1,) * (c.ndim - 1)
        w = _np(a.guidance_b).reshape(shape) if a.guidance_b is not None else f32(a.guidance)
        wu, wc = tw[:, 0].reshape(shape), tw[:, 1].reshape(shape)
        with np.errstate(all="ignore"):
            us = ((u * wu).astype(f32) + (c * wc).astype(f32)).astype(f32)
            g = (us + (w * (c - us)).astype(f32)).astype(f32)
            g = np.where(w == 1, c, g)      # a sample whose scale is 1, per-sample or desc->guidance, gets c
        # the guided raw output is then converted like a single network output
        b = copy.copy(a)
        b.n_model, b.e_cond, b.e_uncond = 1, torch.from_numpy(np.ascontiguousarray(g)), None
        b.guidance_b = b.tcfg_w = None
        b.guidance = 1.0
        return super()._model_value(b, thr)


def guided_net(net, uc, c, w, calls=None):
    """net_g(x, t_input) for a guidance_type="uncond" wrapper: the TCFG output of `net` on cat([x, x]) with cat([uc, c])
    (the words in the device's exact order). `calls`, when a list, receives one entry per network call."""

    def fn(x, t):
        if calls is not None:
            calls.append(tuple(x.shape))
        out_u, out_c = net(torch.cat([x, x]), torch.cat([t, t]), torch.cat([uc, c])).chunk(2)
        words = words_exact(_storage_rows(out_c), _storage_rows(out_u))
        return tcfg_combine(out_c, out_u, words, w)
    return fn
