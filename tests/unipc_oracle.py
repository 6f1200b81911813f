"""Oracles of UniPC sampling (dpm_solver_b200/unipc.py) -- TEST INFRASTRUCTURE.

* `unipc_fp64`: a plain fp64 numpy loop of UniPC multistep as the method is published (Zhao et al. 2023, arXiv:2302.04867,
  the "bh" update of its multistep sampler): predictor, then after the next evaluation the corrector from the same base,
  each step's weights from numpy.linalg.solve. It is written from the formulas, not from dpm_solver_b200/plan.py.
* `words_mp`: the folded fp32 words of every dpm_step_unipc launch, evaluated in mpmath at 50 digits from the same fp32
  marginals the product uses (so that a word can be held to 1 ulp of its exact value).
* `UniPCOracle`: the numpy executor (flow_oracle.FlowOracle, every parameterisation) plus dpm_step_unipc as
  include/dpm_solver_b200.h states it, op for op in IEEE fp32.
"""
import math

import mpmath
import numpy as np
import torch

from flow_oracle import FlowOracle
from oracle_backend import _np, _round

f32 = np.float32


# ---- the method in fp64 ------------------------------------------------------------------------------------------------

def _weights(lam, i, p, data, bh2):
    h = lam[i] - lam[i - 1]
    hh = -h if data else h
    h_phi_1 = math.expm1(hh)
    B = hh if not bh2 else math.expm1(hh)
    r = [(lam[i - 1 - k] - lam[i - 1]) / h for k in range(1, p)] + [1.0]
    R, b = [], []
    h_phi_k = h_phi_1 / hh - 1.0
    f = 1.0
    for j in range(1, p + 1):
        R.append([rk ** (j - 1) for rk in r])
        b.append(h_phi_k * f / B)
        f *= j + 1
        h_phi_k = h_phi_k / hh - 1.0 / f
    R, b = np.array(R), np.array(b)
    rho_p = [] if p == 1 else ([0.5] if p == 2 else list(np.linalg.solve(R[:p - 1, :p - 1], b[:p - 1])))
    rho_c = [0.5] if p == 1 else list(np.linalg.solve(R, b))
    return h_phi_1, B, r, rho_p, rho_c


def orders(N, order, lower_order_final):
    return [min(order, i, N + 1 - i) if lower_order_final else min(order, i) for i in range(1, N + 1)]


def unipc_fp64(model, alpha, sigma, lam, x_T, order, data=True, bh2=True, use_corrector=True,
               lower_order_final=True, return_intermediate=False):
    """model(x, i) -> m_i (x0 when `data`, else eps) at grid point i; alpha, sigma, lam: fp64 sequences over the grid
    t_0 .. t_N. Returns x_N (and the corrected states x_0 .. x_N)."""
    N = len(lam) - 1
    ps = orders(N, order, lower_order_final)
    x = np.asarray(x_T, dtype=np.float64)
    ms = [model(x, 0)]
    xs = [x]
    for i in range(1, N + 1):
        p = ps[i - 1]
        h_phi_1, B, r, rho_p, rho_c = _weights(lam, i, p, data, bh2)
        s = alpha[i] if data else sigma[i]
        a = sigma[i] / sigma[i - 1] if data else alpha[i] / alpha[i - 1]
        D = [(ms[i - 1 - k] - ms[i - 1]) / r[k - 1] for k in range(1, p)]
        base = a * x - s * h_phi_1 * ms[i - 1]
        xt = base - s * B * sum((rho_p[k] * D[k] for k in range(p - 1)), np.zeros_like(x))
        if i == N:
            x = xt
            xs.append(x)
            break
        m = model(xt, i)
        if use_corrector:
            corr = sum((rho_c[k] * D[k] for k in range(p - 1)), np.zeros_like(x)) + rho_c[p - 1] * (m - ms[i - 1])
            x = base - s * B * corr
        else:
            x = xt
        ms.append(m)
        xs.append(x)
    return (x, xs) if return_intermediate else x


# ---- the problem with a closed-form solution ---------------------------------------------------------------------------

class LinearVP64:
    """The continuous linear VP schedule in fp64 (the reference's closed forms, evaluated in double)."""

    def __init__(self, beta_0=0.1, beta_1=20.):
        self.b0, self.b1 = beta_0, beta_1

    def log_alpha(self, t):
        return -0.25 * t ** 2 * (self.b1 - self.b0) - 0.5 * t * self.b0

    def alpha(self, t):
        return math.exp(self.log_alpha(t))

    def sigma(self, t):
        return math.sqrt(1. - math.exp(2. * self.log_alpha(t)))

    def lam(self, t):
        return self.log_alpha(t) - 0.5 * math.log(1. - math.exp(2. * self.log_alpha(t)))

    def inverse_lambda(self, l):
        tmp = 2. * (self.b1 - self.b0) * np.logaddexp(-2. * l, 0.)
        return tmp / (math.sqrt(self.b0 ** 2 + tmp) + self.b0) / (self.b1 - self.b0)

    def logsnr_grid(self, t_T, t_0, N):
        return [self.inverse_lambda(l) for l in np.linspace(self.lam(t_T), self.lam(t_0), N + 1)]


MU, S = 0.5, 0.3


def gaussian_x0(x, alpha, sigma):
    """The exact denoiser of data N(MU, S^2) per element."""
    return MU + alpha * S ** 2 / (alpha ** 2 * S ** 2 + sigma ** 2) * (x - alpha * MU)


def exact_solution(x_T, a_T, s_T, a_e, s_e):
    return a_e * MU + math.sqrt(a_e ** 2 * S ** 2 + s_e ** 2) * (x_T - a_T * MU) / math.sqrt(a_T ** 2 * S ** 2 + s_T ** 2)


def anchor_error(N, order, data=True, bh2=True, use_corrector=True, x_T=1.3, t_T=1., t_0=1e-3):
    """|x_N - exact| of the fp64 transcription on the Gaussian problem, logSNR grid, lower_order_final=False."""
    vp = LinearVP64()
    ts = vp.logsnr_grid(t_T, t_0, N)
    al, sg, lm = [vp.alpha(t) for t in ts], [vp.sigma(t) for t in ts], [vp.lam(t) for t in ts]

    def model(x, i):
        x0 = gaussian_x0(x, al[i], sg[i])
        return x0 if data else (x - al[i] * x0) / sg[i]

    xN = unipc_fp64(model, al, sg, lm, np.array([x_T]), order, data, bh2, use_corrector, lower_order_final=False)
    return abs(float(xN[0]) - exact_solution(x_T, al[0], sg[0], al[-1], sg[-1]))


# ---- the folded words in mpmath ----------------------------------------------------------------------------------------

def words_mp(algorithm_type, variant, lam, alpha, sigma, ords, use_corrector, dps=50):
    """Exact (50-digit) values of every word of launches 1 .. N-1 at the given fp32 marginals (python floats): a list of
    dicts with keys cd0, cd1, ct, a, c0, cp0, cp1 (only those the orders use)."""
    mp = mpmath.mp
    mp.dps = dps
    data, bh2 = algorithm_type == "dpmsolver++", variant == "bh2"
    lam = [mpmath.mpf(v) for v in lam]
    al = [mpmath.mpf(v) for v in alpha]
    sg = [mpmath.mpf(v) for v in sigma]
    N = len(ords)

    def weights(i, p):
        h = lam[i] - lam[i - 1]
        hh = -h if data else h
        h_phi_1 = mpmath.expm1(hh)
        B = mpmath.expm1(hh) if bh2 else hh
        r = [(lam[i - 1 - k] - lam[i - 1]) / h for k in range(1, p)] + [mpmath.mpf(1)]
        R, b = [], []
        h_phi_k, f = h_phi_1 / hh - 1, mpmath.mpf(1)
        for j in range(1, p + 1):
            R.append([rk ** (j - 1) for rk in r])
            b.append(h_phi_k * f / B)
            f *= j + 1
            h_phi_k = h_phi_k / hh - 1 / f
        if p == 1:
            rho_p = []
        elif p == 2:
            rho_p = [mpmath.mpf(1) / 2]
        else:
            rho_p = list(mpmath.lu_solve(mpmath.matrix([row[:2] for row in R[:2]]), mpmath.matrix(b[:2])))
        rho_c = [mpmath.mpf(1) / 2] if p == 1 else list(mpmath.lu_solve(mpmath.matrix(R), mpmath.matrix(b)))
        return h_phi_1, B, r, rho_p, rho_c

    scale = al if data else sg
    out = []
    for i in range(1, N):
        p, q = ords[i - 1], ords[i]
        _, B, r, rho_p, rho_c = weights(i, p)
        w = {}
        if use_corrector:
            for k in range(1, p):
                w["cd%d" % (k - 1)] = -scale[i] * B * (rho_c[k - 1] - rho_p[k - 1]) / r[k - 1]
            w["ct"] = -scale[i] * B * rho_c[p - 1]
        h1, B2, r2, rho_p2, _ = weights(i + 1, q)
        w["a"] = sg[i + 1] / sg[i] if data else al[i + 1] / al[i]
        w["c0"] = -scale[i + 1] * h1
        for k in range(1, q):
            w["cp%d" % (k - 1)] = -scale[i + 1] * B2 * rho_p2[k - 1] / r2[k - 1]
        out.append(w)
    return out


def ulp32(v):
    """Spacing of fp32 at |v| (v an mpmath or python number)."""
    v = abs(float(v))
    return float(np.spacing(f32(v))) if v > 0 else float(np.spacing(f32(0)))


# ---- the executor ------------------------------------------------------------------------------------------------------

class UniPCOracle(FlowOracle):
    """The numpy executor with dpm_step_unipc."""

    def step(self, a):
        if getattr(a, "unipc", None) is None:
            return super().step(a)
        self.launches += 1
        w = a.unipc
        self.log.append(("unipc", a.n_model, w.pc, w.pp))
        ref = a.reference_tensor()
        sdt = a.state_dtype or a.x.dtype
        x = _np(a.x)
        with np.errstate(all="ignore"):
            if a.n_model > 0:
                if a.xe is None:
                    a.xe = a.x
                T = _round(self._model_value(a, _np(a.thr) if a.thr is not None else None), sdt)
            else:
                T = _np(a.m0)
            m1, m2, m3 = _np(a.m1), _np(a.m2), _np(a.m3)
            c = x
            if w.pc > 0:
                if w.pc >= 2:
                    c = c + f32(w.cd[0]) * (m2 - m1)
                if w.pc >= 3:
                    c = c + f32(w.cd[1]) * (m3 - m1)
                c = _round((c + f32(w.ct) * (T - m1)).astype(f32), sdt)
            o = f32(w.a) * c + f32(w.c0) * T
            if w.pp >= 2:
                o = o + f32(w.cp[0]) * (m1 - T)
            if w.pp >= 3:
                o = o + f32(w.cp[1]) * (m2 - T)
        m_out = out = None
        if a.n_model > 0 and a.want_m_out:
            m_out = torch.from_numpy(np.ascontiguousarray(T)).to(sdt).reshape(ref.shape)
        if a.out_c is not None:
            a.out_c.copy_(torch.from_numpy(np.ascontiguousarray(np.asarray(c, dtype=f32))).to(sdt).reshape(a.out_c.shape))
        if w.pp > 0:
            out = torch.from_numpy(np.ascontiguousarray(o.astype(f32))).to(sdt).reshape(ref.shape)
            if a.out is not None:
                a.out.copy_(out.reshape(a.out.shape))
                out = a.out
            if a.out2 is not None:
                a.out2.copy_(out.reshape(a.out2.shape))
        return m_out, out
