"""Oracles of Perp-Neg (model_wrapper's perp_neg) -- TEST INFRASTRUCTURE.

* `perpneg_reference`: the method in float64, written from its formula: with d_k = e_k - u per sample,
  eps = u + s_1*d_1 + sum_{k>=2} s_k*(d_k - (<d_k, d_1>/||d_1||^2)*d_1).
* `sums_exact`: the fp64 sums N = sum d_1*d_1 and P_k = sum d_k*d_1 as the Perp-Neg words pass forms them
  (apg_oracle.device_sum: the chunks, thread ownership, warp butterflies, warp order and chunk merge of words.cu).
* `words_final`: k_perpneg_final's fold of the merged sums, fp64 left to right with each op rounded, rounded to fp32.
* `words_exact`: both together, bit-exact with dpm_perpneg_words; `words_fsum`: the fold on exactly rounded sums.
* `fold_order_case`: blocks whose words differ between the fold's order and its reverse (`words_final_reversed`).
* `PerpNegOracle`: the numpy executor (cfg_mask_oracle.MaskOracle, which serves dpm_step_multi_masked) plus
  dpm_perpneg_words, operation for operation.
* `guided_net`: a network for the UNMODIFIED reference's guidance_type="uncond" wrapper that runs a noise network on
  the (K+1)-fold batch and returns the Perp-Neg noise, combined in eager fp32 torch in the step's order.
"""
import math

import numpy as np
import torch

from apg_oracle import device_sum
from cfg_mask_oracle import MaskOracle
from cfgzero_oracle import _storage_rows

f32 = np.float32
NAN32 = np.array([0x7fffffff], np.uint32).view(np.float32)[0]    # the NaN k_perpneg_final writes


def perpneg_reference(u, es, scales):
    """The Perp-Neg output in float64 from u and the K conditional outputs ([B, ...] arrays), scales s_1..s_K."""
    u = np.asarray(u, np.float64)
    B = u.shape[0]
    d = [np.asarray(e, np.float64) - u for e in es]
    d1 = d[0].reshape(B, -1)
    n2 = (d1 * d1).sum(axis=1)
    out = u + scales[0] * d[0]
    for s, dk in zip(scales[1:], d[1:]):
        coef = np.where(n2 == 0, 0.0, (dk.reshape(B, -1) * d1).sum(axis=1) / np.where(n2 == 0, 1.0, n2))
        out = out + s * (dk - coef.reshape((B,) + (1,) * (u.ndim - 1)) * d[0])
    return out


def _diffs(u, es):
    """d_k = e_k - u in fp64 from fp32 [B, per_sample] rows."""
    u = np.asarray(u, f32).astype(np.float64)
    with np.errstate(all="ignore"):
        return [np.asarray(e, f32).astype(np.float64) - u for e in es]


def sums_exact(u, es):
    """(N, [P_2 .. P_K]) per sample, fp64 [B] each, as the device forms them from [B, per_sample] rows."""
    d = _diffs(u, es)
    with np.errstate(all="ignore"):
        return device_sum(d[0] * d[0]), [device_sum(dk * d[0]) for dk in d[1:]]


def words_final(N, P, scales):
    """fp32 [B] from the merged sums: t = s_1, t = t - s_k*c_k (c_k = P_k/N, 0 when N == 0), NaN for a non-finite
    sum. `scales` are rounded to fp32 and widened, as the host hands them over."""
    N = np.atleast_1d(np.asarray(N, np.float64))
    P = [np.atleast_1d(np.asarray(p, np.float64)) for p in P]
    sig = [float(f32(s)) for s in scales]
    out = np.empty(len(N), f32)
    for b in range(len(N)):
        sums = [float(N[b])] + [float(p[b]) for p in P]
        if not all(math.isfinite(v) for v in sums):
            out[b] = NAN32
            continue
        t = sig[0]
        for s, pk in zip(sig[1:], sums[1:]):
            ck = 0.0 if sums[0] == 0.0 else pk / sums[0]
            t = t - s * ck
        out[b] = f32(t)
    return out


def words_exact(u, es, scales):
    """The words of dpm_perpneg_words from [B, per_sample] rows in storage order."""
    return words_final(*sums_exact(u, es), scales)


def words_fsum(u, es, scales):
    """The fold on exactly rounded sums (math.fsum) of the same fp64 products."""
    d = _diffs(u, es)
    N = [math.fsum(r) for r in d[0] * d[0]]
    P = [[math.fsum(r) for r in dk * d[0]] for dk in d[1:]]
    return words_final(N, P, scales)


class PerpNegOracle(MaskOracle):
    """The numpy executor with dpm_perpneg_words (in the device's order, so its words are bit-exact)."""

    def perpneg_words(self, e_uncond, e_conds, scales):
        self.launches += 2
        self.log.append(("perpneg_words", len(e_conds)))
        u = _storage_rows(e_uncond)
        es = [_storage_rows(e, e_uncond) for e in e_conds]
        return torch.from_numpy(words_exact(u, es, scales))


def perp_combine(eu, ecs, scales, w1):
    """eps_u + w1*(eps_1 - eps_u) + s_2*(eps_2 - eps_u) + ... in eager fp32 torch, left to right (w1: fp32 [B])."""
    w = torch.as_tensor(w1).reshape((-1,) + (1,) * (eu.dim() - 1))
    e = eu + w * (ecs[0] - eu)
    for s, ek in zip(scales[1:], ecs[1:]):
        e = e + float(f32(s)) * (ek - eu)
    return e


def guided_net(net, uc, conds, scales, calls=None):
    """net_g(x, t_input) for a guidance_type="uncond" wrapper of a NOISE network: `net` on cat([x] * (K+1)) with
    cat([uc, c_1, ..., c_K]), then the Perp-Neg combine of its blocks with the device's words. `calls`, when a list,
    receives one entry per network call."""
    K = len(conds)

    def fn(x, t):
        if calls is not None:
            calls.append(tuple(x.shape))
        outs = net(torch.cat([x] * (K + 1)), torch.cat([t] * (K + 1)), torch.cat([uc, *conds])).chunk(K + 1)
        w1 = words_exact(_storage_rows(outs[0]), [_storage_rows(o, outs[0]) for o in outs[1:]], scales)
        return perp_combine(outs[0], outs[1:], scales, torch.from_numpy(w1))
    return fn


def words_final_reversed(N, P, scales):
    """words_final with the terms s_k*c_k subtracted from s_1 last to first: the fold order a wrong kernel would use."""
    return words_final(N, P[::-1], [scales[0]] + list(scales[1:])[::-1])


def fold_order_case(B=16, D=96, seed=0):
    """(u, [e_1 .. e_4], scales) as fp32 [B, D] arrays whose words expose the order of the fp64 fold. The blocks sit on
    grids where every difference, product and sum is exact: d_2 = 2^13*d_1 and d_4 = -2^13*d_1, so c_2 = 2^13 and
    c_4 = -2^13 exactly, and with s_2 = s_4 = 2^27 the terms s_2*c_2 = 2^40 and s_4*c_4 = -2^40 cancel exactly; d_3 is
    noise, so s_3*c_3 is of order 1 with every fraction bit set. Folded first to last, t passes just below 2^40 (fp64
    grid 2^-13) while s_1 and s_3*c_3 are pending; folded last to first, it passes just above 2^40 (grid 2^-12). The
    two orders then round t differently by up to 2^-13 -- hundreds of fp32 ulps of a t near 1."""
    rng = np.random.default_rng(seed)
    u = (rng.integers(-4096, 4096, (B, D)) / 1024.0)
    d1 = rng.choice([-8, -5, -3, -1, 1, 2, 4, 7], (B, D)) / 16.0
    d3 = rng.integers(-4096, 4096, (B, D)) / 1024.0
    es = [u + d1, u + 8192.0 * d1, u + d3, u - 8192.0 * d1]
    assert all(np.array_equal(e.astype(f32).astype(np.float64), e) for e in [u] + es)
    return u.astype(f32), [e.astype(f32) for e in es], [1.3, 2.0 ** 27, 1.7, 2.0 ** 27]
