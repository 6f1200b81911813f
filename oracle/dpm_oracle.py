"""CPU oracle for the DPM-Solver update path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A numpy (or, optionally, torch-CPU) restatement of the algorithm of
the reference dpm_solver_pytorch.py for the hot path of SURVEY.md section 8: schedule scalars,
parameterisation / CFG / eps->x0 / dynamic thresholding, the five update formulas and the
multistep / singlestep sampling loops. Every function cites the reference lines it follows.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline leg may import this module. The
product (dpm_solver_b200/) never does: it has no CPU path at all.

Parity pin: the reference ships no tests or golden vectors (SURVEY.md section 4), so this oracle is
pinned against outputs of the reference itself, generated in the build container by
tests/golden/make_golden.py and committed under tests/golden/*.npz (tests/test_oracle_golden.py).

Array namespace: `NP` (numpy, default: independent arithmetic; transcendental scalars may differ
from torch by an ulp) or `TH` (torch CPU: the same ATen kernels the reference runs, used for the
multi-threaded CPU baseline in bench.py). All scalars are fp32 arrays of shape (1,), like the
reference's (1,)-shaped coefficient tensors, so promotion and rounding follow the same rules.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np


# ---------------------------------------------------------------------------------------------
# array namespaces
# ---------------------------------------------------------------------------------------------
class _NP:
    name = "numpy"
    f32 = np.float32

    @staticmethod
    def asarray(v, dtype=np.float32):
        return np.asarray(v, dtype=dtype)

    exp = staticmethod(np.exp)
    log = staticmethod(np.log)
    sqrt = staticmethod(np.sqrt)
    expm1 = staticmethod(np.expm1)
    logaddexp = staticmethod(np.logaddexp)
    abs = staticmethod(np.abs)
    maximum = staticmethod(np.maximum)

    @staticmethod
    def clip(x, lo, hi):
        return np.minimum(np.maximum(x, lo), hi)

    @staticmethod
    def linspace(a, b, n):
        # torch.linspace(dtype=float32) on CPU: fp32 endpoints and fp32 step, each point is the
        # fused multiply-add start + step*i (end - step*(n-1-i) in the upper half)
        a32, b32 = np.float32(a), np.float32(b)
        if n == 1:
            return np.array([a32], dtype=np.float32)
        step = np.float64(np.float32((b32 - a32) / np.float32(n - 1)))
        i = np.arange(n)
        lo = (np.float64(a32) + step * i).astype(np.float32)
        hi = (np.float64(b32) - step * (n - 1 - i)).astype(np.float32)
        return np.where(i < n // 2, lo, hi)

    @staticmethod
    def cat(xs):
        return np.concatenate(xs)

    @staticmethod
    def sort_with_index(a):
        idx = np.argsort(a, kind="stable")
        return a[idx], idx

    @staticmethod
    def flip(a):
        return a[::-1].copy()

    @staticmethod
    def zeros1():
        return np.zeros((1,), dtype=np.float32)

    @staticmethod
    def reshape(a, shape):
        return np.reshape(a, shape)


NP = _NP()


def _torch_ns(device="cpu"):
    import torch

    class _TH:
        name = "torch"
        f32 = torch.float32

        @staticmethod
        def asarray(v, dtype=torch.float32):
            return torch.as_tensor(v, dtype=dtype, device=device)

        exp, log, sqrt, expm1 = torch.exp, torch.log, torch.sqrt, torch.expm1
        logaddexp, abs, maximum = torch.logaddexp, torch.abs, torch.maximum

        @staticmethod
        def clip(x, lo, hi):
            return torch.clamp(x, lo, hi)

        @staticmethod
        def linspace(a, b, n):
            return torch.linspace(a, b, n).to(device)     # the reference builds grids on CPU, then .to(device) (:474)

        @staticmethod
        def cat(xs):
            return torch.cat(xs)

        @staticmethod
        def sort_with_index(a):
            return torch.sort(a)

        @staticmethod
        def flip(a):
            return torch.flip(a, [0])

        @staticmethod
        def zeros1():
            return torch.zeros((1,), device=device)

        @staticmethod
        def reshape(a, shape):
            return a.reshape(shape)

    return _TH()


def torch_namespace(device="cpu"):
    """torch ops on `device`: 'cpu' = the CPU baseline; 'cuda' = the reference algorithm as stock eager
    PyTorch CUDA kernels (every scalar op a launch, every update 3/7/16 full-tensor launches)."""
    return _torch_ns(device)


def _scalar(xp, v):
    """fp32 array of shape (1,) (the reference's coefficient tensors have this shape)."""
    if isinstance(v, (int, float)):
        return xp.asarray([v])
    return xp.reshape(v, (-1,))


# ---------------------------------------------------------------------------------------------
# NoiseScheduleVP (reference :6-167) and interpolate_fn (:1253-1292)
# ---------------------------------------------------------------------------------------------
def _interpolate_tensor_ops(x, kx, ky):
    """torch namespace: interpolate_fn as a chain of tensor ops without host control flow, the way the
    reference runs it on a device (cat, sort, argmin, where, gather :1266-1291) -- one launch per op."""
    import torch
    n, K = x.shape[0], kx.shape[0]
    both = torch.cat([x.reshape(n, 1), kx.reshape(1, K).repeat(n, 1)], dim=1)      # :1267
    srt, order = torch.sort(both, dim=1)                                             # :1268
    pos = torch.argmin(order, dim=1)                                                 # :1269
    below = pos - 1
    one = torch.tensor(1, device=x.device)
    last = torch.tensor(K - 2, device=x.device)
    start = torch.where(torch.eq(pos, 0), one, torch.where(torch.eq(pos, K), last, below))        # :1271-1277
    end = torch.where(torch.eq(start, below), start + 2, start + 1)                               # :1278
    x0 = torch.gather(srt, 1, start.unsqueeze(1)).squeeze(1)                                     # :1279
    x1 = torch.gather(srt, 1, end.unsqueeze(1)).squeeze(1)                                       # :1280
    s2 = torch.where(torch.eq(pos, 0), torch.tensor(0, device=x.device), torch.where(torch.eq(pos, K), last, below))  # :1281-1287
    kyb = ky.reshape(1, K).expand(n, -1)                                                          # :1288
    y0 = torch.gather(kyb, 1, s2.unsqueeze(1)).squeeze(1)                                        # :1289
    y1 = torch.gather(kyb, 1, (s2 + 1).unsqueeze(1)).squeeze(1)                                  # :1290
    return y0 + (x - x0) * (y1 - y0) / (x1 - x0)                                                 # :1291


def interpolate(xp, x, kx, ky):
    """Piecewise-linear f(x) through keypoints (kx, ky), linear extrapolation outside.

    Follows interpolate_fn :1266-1291 literally, one query at a time: sort the query together with
    the keypoints (query first), locate it, pick the bracketing keypoints, then
    y0 + (x - x0) * (y1 - y0) / (x1 - x0)."""
    if xp.name == "torch":
        return _interpolate_tensor_ops(x, kx, ky)
    K = kx.shape[0]
    out = []
    for q in range(x.shape[0]):
        xq = x[q:q + 1]
        both = xp.cat([xq, kx])                       # :1267
        srt, idx = xp.sort_with_index(both)           # :1268
        pos = int((idx == 0).nonzero()[0][0]) if xp.name == "numpy" else int((idx == 0).nonzero()[0])  # :1269
        if pos == 0:                                  # :1271-1277
            start = 1
        elif pos == K:
            start = K - 2
        else:
            start = pos - 1
        end = start + 2 if start == pos - 1 else start + 1   # :1278
        x0, x1 = srt[start:start + 1], srt[end:end + 1]      # :1279-1280
        if pos == 0:                                  # :1281-1287
            s2 = 0
        elif pos == K:
            s2 = K - 2
        else:
            s2 = pos - 1
        y0, y1 = ky[s2:s2 + 1], ky[s2 + 1:s2 + 2]     # :1288-1290
        out.append(y0 + (xq - x0) * (y1 - y0) / (x1 - x0))   # :1291
    return xp.cat(out)


class VPSchedule:
    """NoiseScheduleVP (:6-167): 'discrete' (table of log alpha) or 'linear' (continuous VPSDE)."""

    def __init__(self, schedule="discrete", log_alpha_table=None, total_N=None, beta_0=0.1, beta_1=20.,
                 xp=NP):
        if schedule not in ("discrete", "linear"):
            raise ValueError("unsupported schedule")
        self.schedule, self.xp, self.T = schedule, xp, 1.0
        if schedule == "discrete":
            self.log_alpha = xp.asarray(log_alpha_table)          # already clipped (:105)
            self.total_N = int(self.log_alpha.shape[0])           # :106
            self.t = xp.linspace(0., 1., self.total_N + 1)[1:]    # :107
        else:
            self.total_N, self.beta_0, self.beta_1 = 1000, beta_0, beta_1              # :110-112

    @classmethod
    def from_betas(cls, betas64, xp=NP):
        """log_alphas = 0.5*cumsum(log(1-betas)) (:100), then numerical_clip_alpha (:114-125)."""
        betas64 = np.asarray(betas64, dtype=np.float64)
        log_alphas = 0.5 * np.cumsum(np.log(1 - betas64))
        log_sigmas = 0.5 * np.log(1. - np.exp(2. * log_alphas))
        lambs = log_alphas - log_sigmas
        idx = int(np.searchsorted(lambs[::-1], -5.1))
        if idx > 0:
            log_alphas = log_alphas[:-idx]
        return cls("discrete", log_alpha_table=log_alphas.astype(np.float32), xp=xp)

    def set_tables(self, t_table, log_alpha_table):
        """Use the exact fp32 tables of a reference instance (pins table construction separately)."""
        self.t, self.log_alpha = self.xp.asarray(t_table), self.xp.asarray(log_alpha_table)
        self.total_N = int(self.log_alpha.shape[0])

    def marginal_log_mean_coeff(self, t):     # :127-134
        t = _scalar(self.xp, t)
        if self.schedule == "discrete":
            return interpolate(self.xp, t, self.t, self.log_alpha)
        return -0.25 * t ** 2 * (self.beta_1 - self.beta_0) - 0.5 * t * self.beta_0

    def marginal_alpha(self, t):              # :136-140
        return self.xp.exp(self.marginal_log_mean_coeff(t))

    def marginal_std(self, t):                # :142-146
        return self.xp.sqrt(1. - self.xp.exp(2. * self.marginal_log_mean_coeff(t)))

    def marginal_lambda(self, t):             # :148-154
        lmc = self.marginal_log_mean_coeff(t)
        log_std = 0.5 * self.xp.log(1. - self.xp.exp(2. * lmc))
        return lmc - log_std

    def inverse_lambda(self, lamb):           # :156-167
        xp = self.xp
        lamb = _scalar(xp, lamb)
        if self.schedule == "linear":
            tmp = 2. * (self.beta_1 - self.beta_0) * xp.logaddexp(-2. * lamb, xp.zeros1())
            Delta = self.beta_0 ** 2 + tmp
            return tmp / (xp.sqrt(Delta) + self.beta_0) / (self.beta_1 - self.beta_0)
        log_alpha = -0.5 * xp.logaddexp(xp.zeros1(), -2. * lamb)
        return interpolate(xp, log_alpha, xp.flip(self.log_alpha), xp.flip(self.t))


# ---------------------------------------------------------------------------------------------
# model_wrapper pieces (:271-330) and data prediction (:416-442)
# ---------------------------------------------------------------------------------------------
def model_input_time(ns, t):                       # :271-280
    if ns.schedule == "discrete":
        return (t - 1. / ns.total_N) * 1000.
    return t


def to_noise(ns, model_type, x, out, t):           # noise_pred_fn :288-298
    if model_type == "noise":
        return out
    if model_type == "x_start":
        return (x - ns.marginal_alpha(t) * out) / ns.marginal_std(t)
    if model_type == "v":
        return ns.marginal_alpha(t) * out + ns.marginal_std(t) * x
    if model_type == "score":
        return -ns.marginal_std(t) * out
    raise ValueError(model_type)


def cfg_combine(eps_uncond, eps_cond, scale):      # model_fn :330
    return eps_uncond + scale * (eps_cond - eps_uncond)


def _fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c): exact rationals for finite operands, IEEE semantics otherwise.

    With an infinite or NaN operand the result is inf or NaN, and float64 arithmetic gives the IEEE one: the
    product of two fp32 values is exact there, inf * 0 and inf - inf are NaN. A finite result beyond the fp32
    range rounds to inf, which takes part in round-to-nearest-even as 2^128 with an even significand."""
    a, b, c = np.float32(a), np.float32(b), np.float32(c)
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        with np.errstate(invalid="ignore", over="ignore"):
            return np.float32(np.float64(a) * np.float64(b) + np.float64(c))
    r = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    with np.errstate(over="ignore"):
        f = np.float32(float(r))
        cands = {float(f), float(np.nextafter(f, np.float32(np.inf))), float(np.nextafter(f, np.float32(-np.inf)))}
    best = None
    for cnd in cands:
        if math.isnan(cnd):
            continue
        v = Fraction(cnd) if math.isfinite(cnd) else Fraction(2 ** 128) * (1 if cnd > 0 else -1)
        d = abs(v - r)
        even = (np.float32(cnd).view(np.uint32) & 1) == 0
        key = (d, 0 if even else 1)
        if best is None or key < best[0]:
            best = (key, cnd)
    return np.float32(best[1])


def quantile_abs(x0, q):
    """torch.quantile(|x0|.reshape(B,-1), q, dim=1) (:422): sort, fp32 rank q*(n-1), lerp between the
    two adjacent order statistics with ATen's CPU lerp: fma(w<0.5 ? w : w-1, hi-lo, w<0.5 ? lo : hi).
    Non-finite order statistics follow torch: inf - inf in the lerp gives NaN, a NaN in the row gives NaN."""
    a = np.abs(np.asarray(x0, dtype=np.float32)).reshape(x0.shape[0], -1)
    n = a.shape[1]
    srt = np.sort(a, axis=1)
    pos = np.float32(q) * np.float32(n - 1)
    lo = int(np.floor(pos))
    hi = int(np.ceil(pos))
    w = np.float32(pos - np.float32(lo))
    out = np.empty((a.shape[0],), dtype=np.float32)
    for b in range(a.shape[0]):
        if np.isnan(srt[b, -1]):          # numpy sorts NaN last; torch.quantile returns NaN when the row holds one
            out[b] = np.float32(np.nan)
            continue
        vl, vh = srt[b, lo], srt[b, min(hi, n - 1)]
        with np.errstate(invalid="ignore"):
            d = np.float32(vh - vl)
        out[b] = _fma32(w, d, vl) if w < np.float32(0.5) else _fma32(np.float32(w - np.float32(1)), d, vh)
    return out


def dynamic_thresholding(x0, ratio=0.995, max_val=1.0):    # :416-425
    x0 = np.asarray(x0, dtype=np.float32)
    s = np.maximum(quantile_abs(x0, ratio), np.float32(max_val))          # :422-423
    s = s.reshape((-1,) + (1,) * (x0.ndim - 1))
    return (np.minimum(np.maximum(x0, -s), s) / s).astype(np.float32)    # :424


def data_prediction(ns, x, noise, t, thresholding=None):   # :433-442
    alpha_t, sigma_t = ns.marginal_alpha(t), ns.marginal_std(t)
    x0 = (x - sigma_t * noise) / alpha_t
    if thresholding is not None:
        x0 = dynamic_thresholding(x0, *thresholding)
    return x0


# ---------------------------------------------------------------------------------------------
# the five update formulas
# ---------------------------------------------------------------------------------------------
def first_update(ns, algo, x, s, t, model_s):              # :561-588
    xp = ns.xp
    h = ns.marginal_lambda(t) - ns.marginal_lambda(s)
    if algo == "dpmsolver++":
        phi_1 = xp.expm1(-h)
        return ns.marginal_std(t) / ns.marginal_std(s) * x - xp.exp(ns.marginal_log_mean_coeff(t)) * phi_1 * model_s
    phi_1 = xp.expm1(h)
    return (xp.exp(ns.marginal_log_mean_coeff(t) - ns.marginal_log_mean_coeff(s)) * x
            - (ns.marginal_std(t) * phi_1) * model_s)


def multistep_second(ns, algo, solver_type, x, models, times, t):   # :812-852; lists oldest -> newest
    xp = ns.xp
    m1, m0 = models[-2], models[-1]
    t1, t0 = times[-2], times[-1]
    l1, l0, lt = ns.marginal_lambda(t1), ns.marginal_lambda(t0), ns.marginal_lambda(t)
    la0, lat = ns.marginal_log_mean_coeff(t0), ns.marginal_log_mean_coeff(t)
    sg0, sgt = ns.marginal_std(t0), ns.marginal_std(t)
    alpha_t = xp.exp(lat)
    h_0, h = l0 - l1, lt - l0
    r0 = h_0 / h
    D1_0 = (1. / r0) * (m0 - m1)
    if algo == "dpmsolver++":
        phi_1 = xp.expm1(-h)
        if solver_type == "dpmsolver":
            return (sgt / sg0) * x - (alpha_t * phi_1) * m0 - 0.5 * (alpha_t * phi_1) * D1_0
        return (sgt / sg0) * x - (alpha_t * phi_1) * m0 + (alpha_t * (phi_1 / h + 1.)) * D1_0
    phi_1 = xp.expm1(h)
    if solver_type == "dpmsolver":
        return xp.exp(lat - la0) * x - (sgt * phi_1) * m0 - 0.5 * (sgt * phi_1) * D1_0
    return xp.exp(lat - la0) * x - (sgt * phi_1) * m0 - (sgt * (phi_1 / h - 1.)) * D1_0


def multistep_third(ns, algo, x, models, times, t):        # :868-904
    xp = ns.xp
    m2, m1, m0 = models
    t2, t1, t0 = times
    l2, l1, l0, lt = (ns.marginal_lambda(v) for v in (t2, t1, t0, t))
    la0, lat = ns.marginal_log_mean_coeff(t0), ns.marginal_log_mean_coeff(t)
    sg0, sgt = ns.marginal_std(t0), ns.marginal_std(t)
    alpha_t = xp.exp(lat)
    h_1, h_0, h = l1 - l2, l0 - l1, lt - l0
    r0, r1 = h_0 / h, h_1 / h
    D1_0 = (1. / r0) * (m0 - m1)
    D1_1 = (1. / r1) * (m1 - m2)
    D1 = D1_0 + (r0 / (r0 + r1)) * (D1_0 - D1_1)
    D2 = (1. / (r0 + r1)) * (D1_0 - D1_1)
    if algo == "dpmsolver++":
        phi_1 = xp.expm1(-h)
        phi_2 = phi_1 / h + 1.
        phi_3 = phi_2 / h - 0.5
        return (sgt / sg0) * x - (alpha_t * phi_1) * m0 + (alpha_t * phi_2) * D1 - (alpha_t * phi_3) * D2
    phi_1 = xp.expm1(h)
    phi_2 = phi_1 / h - 1.
    phi_3 = phi_2 / h - 0.5
    return xp.exp(lat - la0) * x - (sgt * phi_1) * m0 - (sgt * phi_2) * D1 - (sgt * phi_3) * D2


def singlestep_second(ns, algo, solver_type, x, s, t, model_fn, r1=0.5, model_s=None):   # :613-673
    xp = ns.xp
    if r1 is None:
        r1 = 0.5
    ls, lt = ns.marginal_lambda(s), ns.marginal_lambda(t)
    h = lt - ls
    s1 = ns.inverse_lambda(ls + r1 * h)
    las, la1, lat = (ns.marginal_log_mean_coeff(v) for v in (s, s1, t))
    sgs, sg1, sgt = (ns.marginal_std(v) for v in (s, s1, t))
    al1, alt = xp.exp(la1), xp.exp(lat)
    if model_s is None:
        model_s = model_fn(x, s)
    if algo == "dpmsolver++":
        phi_11, phi_1 = xp.expm1(-r1 * h), xp.expm1(-h)
        x_s1 = (sg1 / sgs) * x - (al1 * phi_11) * model_s
        model_s1 = model_fn(x_s1, s1)
        if solver_type == "dpmsolver":
            x_t = (sgt / sgs) * x - (alt * phi_1) * model_s - (0.5 / r1) * (alt * phi_1) * (model_s1 - model_s)
        else:
            x_t = (sgt / sgs) * x - (alt * phi_1) * model_s + (1. / r1) * (alt * (phi_1 / h + 1.)) * (model_s1 - model_s)
    else:
        phi_11, phi_1 = xp.expm1(r1 * h), xp.expm1(h)
        x_s1 = xp.exp(la1 - las) * x - (sg1 * phi_11) * model_s
        model_s1 = model_fn(x_s1, s1)
        if solver_type == "dpmsolver":
            x_t = xp.exp(lat - las) * x - (sgt * phi_1) * model_s - (0.5 / r1) * (sgt * phi_1) * (model_s1 - model_s)
        else:
            x_t = xp.exp(lat - las) * x - (sgt * phi_1) * model_s - (1. / r1) * (sgt * (phi_1 / h - 1.)) * (model_s1 - model_s)
    return x_t, {"model_s": model_s, "model_s1": model_s1}


def singlestep_third(ns, algo, solver_type, x, s, t, model_fn, r1=1. / 3., r2=2. / 3., model_s=None,
                     model_s1=None):                                                       # :697-794
    xp = ns.xp
    if r1 is None:
        r1 = 1. / 3.
    if r2 is None:
        r2 = 2. / 3.
    ls, lt = ns.marginal_lambda(s), ns.marginal_lambda(t)
    h = lt - ls
    s1, s2 = ns.inverse_lambda(ls + r1 * h), ns.inverse_lambda(ls + r2 * h)
    las, la1, la2, lat = (ns.marginal_log_mean_coeff(v) for v in (s, s1, s2, t))
    sgs, sg1, sg2, sgt = (ns.marginal_std(v) for v in (s, s1, s2, t))
    al1, al2, alt = xp.exp(la1), xp.exp(la2), xp.exp(lat)
    if model_s is None:
        model_s = model_fn(x, s)
    if algo == "dpmsolver++":
        phi_11, phi_12, phi_1 = xp.expm1(-r1 * h), xp.expm1(-r2 * h), xp.expm1(-h)
        phi_22 = xp.expm1(-r2 * h) / (r2 * h) + 1.
        phi_2 = phi_1 / h + 1.
        phi_3 = phi_2 / h - 0.5
        if model_s1 is None:
            x_s1 = (sg1 / sgs) * x - (al1 * phi_11) * model_s
            model_s1 = model_fn(x_s1, s1)
        x_s2 = (sg2 / sgs) * x - (al2 * phi_12) * model_s + r2 / r1 * (al2 * phi_22) * (model_s1 - model_s)
        model_s2 = model_fn(x_s2, s2)
        if solver_type == "dpmsolver":
            x_t = (sgt / sgs) * x - (alt * phi_1) * model_s + (1. / r2) * (alt * phi_2) * (model_s2 - model_s)
        else:
            D1_0 = (1. / r1) * (model_s1 - model_s)
            D1_1 = (1. / r2) * (model_s2 - model_s)
            D1 = (r2 * D1_0 - r1 * D1_1) / (r2 - r1)
            D2 = 2. * (D1_1 - D1_0) / (r2 - r1)
            x_t = (sgt / sgs) * x - (alt * phi_1) * model_s + (alt * phi_2) * D1 - (alt * phi_3) * D2
    else:
        phi_11, phi_12, phi_1 = xp.expm1(r1 * h), xp.expm1(r2 * h), xp.expm1(h)
        phi_22 = xp.expm1(r2 * h) / (r2 * h) - 1.
        phi_2 = phi_1 / h - 1.
        phi_3 = phi_2 / h - 0.5
        if model_s1 is None:
            x_s1 = xp.exp(la1 - las) * x - (sg1 * phi_11) * model_s
            model_s1 = model_fn(x_s1, s1)
        x_s2 = xp.exp(la2 - las) * x - (sg2 * phi_12) * model_s - r2 / r1 * (sg2 * phi_22) * (model_s1 - model_s)
        model_s2 = model_fn(x_s2, s2)
        if solver_type == "dpmsolver":
            x_t = xp.exp(lat - las) * x - (sgt * phi_1) * model_s - (1. / r2) * (sgt * phi_2) * (model_s2 - model_s)
        else:
            D1_0 = (1. / r1) * (model_s1 - model_s)
            D1_1 = (1. / r2) * (model_s2 - model_s)
            D1 = (r2 * D1_0 - r1 * D1_1) / (r2 - r1)
            D2 = 2. * (D1_1 - D1_0) / (r2 - r1)
            x_t = xp.exp(lat - las) * x - (sgt * phi_1) * model_s - (sgt * phi_2) * D1 - (sgt * phi_3) * D2
    return x_t, {"model_s": model_s, "model_s1": model_s1, "model_s2": model_s2}


# ---------------------------------------------------------------------------------------------
# time grids and sampling loops (:453-539, :1171-1241)
# ---------------------------------------------------------------------------------------------
def time_steps(ns, skip_type, t_T, t_0, N):            # :453-480
    xp = ns.xp
    if skip_type == "logSNR":
        lam_T = ns.marginal_lambda(xp.asarray([t_T]))
        lam_0 = ns.marginal_lambda(xp.asarray([t_0]))
        return ns.inverse_lambda(xp.linspace(float(lam_T[0]), float(lam_0[0]), N + 1))
    if skip_type == "time_uniform":
        return xp.linspace(t_T, t_0, N + 1)
    if skip_type == "time_quadratic":
        return xp.linspace(t_T ** 0.5, t_0 ** 0.5, N + 1) ** 2
    raise ValueError(skip_type)


def singlestep_orders(steps, order):                   # :514-533
    if order == 3:
        K = steps // 3 + 1
        rem = steps % 3
        return [3] * (K - 2) + [2, 1] if rem == 0 else [3] * (K - 1) + ([1] if rem == 1 else [2])
    if order == 2:
        return [2] * (steps // 2) + ([1] if steps % 2 else [])
    if order == 1:
        return [1] * steps
    raise ValueError("'order' must be '1' or '2' or '3'.")


class Sampler:
    """DPM_Solver.sample() for method in {multistep, singlestep, singlestep_fixed} (:1171-1241).

    `net(x, t_in)` is the raw network (numpy in / numpy out, or torch with xp=TH); `model_type`,
    CFG (`guidance_scale`, with the network then receiving a doubled batch, unconditional half
    first :326-329) and dynamic thresholding follow the reference."""

    def __init__(self, ns, net, algorithm_type="dpmsolver++", model_type="noise", guidance_scale=None,
                 thresholding=None):
        self.ns, self.net, self.algo = ns, net, algorithm_type
        self.model_type, self.scale, self.thr = model_type, guidance_scale, thresholding
        self.calls = []   # (t_in[0], x.shape) per network call
        self.log_calls = True   # reading t_in[0] syncs a device; timing runs switch it off

    def noise(self, x, t):                              # model_fn :309-330 + self.model :404
        xp = self.ns.xp
        B = x.shape[0]
        t1 = _scalar(xp, t)[0:1]                        # one time label for the whole batch (:404)
        if self.scale is None:
            t_in = model_input_time(self.ns, xp.cat([t1] * B))
            if self.log_calls:
                self.calls.append((float(t_in[0]), tuple(x.shape)))
            return to_noise(self.ns, self.model_type, x, self.net(x, t_in), t1)
        x2 = xp.cat([x, x])                             # :326
        t_in = model_input_time(self.ns, xp.cat([t1] * (2 * B)))   # :327
        if self.log_calls:
            self.calls.append((float(t_in[0]), tuple(x2.shape)))
        if self.scale == 1.:
            # :323-324: a scale of exactly 1 bypasses the combine -- the reference evaluates the conditional
            # branch alone. This two-argument `net` only reaches that branch through the doubled batch, so
            # the batch is still doubled here and the conditional half returned unchanged (same values for
            # a per-sample network); the call is logged with the shape the reference's single call has.
            if self.log_calls:
                self.calls[-1] = (float(t_in[0]), tuple(x.shape))
            return to_noise(self.ns, self.model_type, x2, self.net(x2, t_in), t1)[B:]
        both = to_noise(self.ns, self.model_type, x2, self.net(x2, t_in), t1)
        return cfg_combine(both[:B], both[B:], self.scale)          # :329-330, uncond half first

    def model_fn(self, x, t):                           # :444-451
        eps = self.noise(x, t)
        if self.algo == "dpmsolver++":
            return data_prediction(self.ns, x, eps, t, self.thr)
        return eps

    def multistep(self, x, steps, order, skip_type="time_uniform", t_T=None, t_0=None,
                  lower_order_final=True, solver_type="dpmsolver"):
        ns = self.ns
        t_0 = 1. / ns.total_N if t_0 is None else t_0
        t_T = ns.T if t_T is None else t_T
        ts = time_steps(ns, skip_type, t_T, t_0, steps)
        inter = []
        tp = [ts[0:1]]
        mp = [self.model_fn(x, ts[0:1])]
        inter.append(x)
        for step in range(1, order):                    # :1185-1193
            x = self._ms_update(x, mp, tp, ts[step:step + 1], step, solver_type)
            inter.append(x)
            tp.append(ts[step:step + 1])
            mp.append(self.model_fn(x, ts[step:step + 1]))
        for step in range(order, steps + 1):            # :1195-1213
            so = min(order, steps + 1 - step) if (lower_order_final and steps < 10) else order
            x = self._ms_update(x, mp, tp, ts[step:step + 1], so, solver_type)
            inter.append(x)
            for i in range(order - 1):
                tp[i], mp[i] = tp[i + 1], mp[i + 1]
            tp[-1] = ts[step:step + 1]
            if step < steps:
                mp[-1] = self.model_fn(x, ts[step:step + 1])
        return x, inter

    def _ms_update(self, x, mp, tp, t, order, solver_type):          # :947-954
        if order == 1:
            return first_update(self.ns, self.algo, x, tp[-1], t, mp[-1])
        if order == 2:
            return multistep_second(self.ns, self.algo, solver_type, x, mp, tp, t)
        if order == 3:
            return multistep_third(self.ns, self.algo, x, mp, tp, t)
        raise ValueError(order)

    def singlestep(self, x, steps, order, skip_type="time_uniform", t_T=None, t_0=None,
                   solver_type="dpmsolver", fixed=False):
        ns, xp = self.ns, self.ns.xp
        t_0 = 1. / ns.total_N if t_0 is None else t_0
        t_T = ns.T if t_T is None else t_T
        if fixed:                                       # :1217-1220
            K = steps // order
            orders = [order] * K
            outer = time_steps(ns, skip_type, t_T, t_0, K)
        else:                                           # :534-538
            orders = singlestep_orders(steps, order)
            if skip_type == "logSNR":
                outer = time_steps(ns, skip_type, t_T, t_0, len(orders))
            else:
                full = time_steps(ns, skip_type, t_T, t_0, steps)
                outer = full[np.cumsum([0] + orders)]
        inter = []
        for step, o in enumerate(orders):               # :1221-1232
            s, t = outer[step:step + 1], outer[step + 1:step + 2]
            inner = time_steps(ns, skip_type, float(s[0]), float(t[0]), o)
            lam = ns.marginal_lambda(inner)
            h = lam[-1:] - lam[0:1]
            r1 = None if o <= 1 else (lam[1:2] - lam[0:1]) / h
            r2 = None if o <= 2 else (lam[2:3] - lam[0:1]) / h
            if o == 1:
                x = first_update(ns, self.algo, x, s, t, self.model_fn(x, s))
            elif o == 2:
                x, _ = singlestep_second(ns, self.algo, solver_type, x, s, t, self.model_fn, r1)
            else:
                x, _ = singlestep_third(ns, self.algo, solver_type, x, s, t, self.model_fn, r1, r2)
            inter.append(x)
        return x, inter
