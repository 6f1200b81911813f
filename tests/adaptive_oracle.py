"""Oracle of the device step-size controller of dpm_solver_adaptive (csrc/adaptive_ctl.cu), CPU only.

The controller's contract is the reference's fp32 arithmetic, op for op (dpm_solver_pytorch.py:156-166, :972-1008),
with exp / log / expm1 / log1p correctly rounded to fp32 and float_power(E, -1/order) taken as the exact power
rounded to fp64 and then to fp32 (the reference's own double rounding). sqrt is correctly rounded too, as IEEE and
the device's sqrtf have it; torch's CPU sqrt is not (one ulp off on ~0.5 % of fp32 arguments). This module evaluates
exactly that:

  * the scalars come from plan.py / schedule.py -- bit-identical to the reference on the CPU (test_host_logic.py) --
    and from the host controller's update (solver.py, dpm_solver_adaptive), run inside `libm()`, a context that
    replaces torch.exp / log / expm1 / log1p / sqrt / logaddexp / float_power by elementwise versions from mpmath
    at PREC bits and rounded once (logaddexp rebuilt as ATen computes it: max + log1p(exp(-|a - b|)));
  * `init`, `plan` and `decide` return every word the three kernels write: state[16] (integral words as int bit
    patterns), coef[4][16] (11 live words per block; the others keep what the caller passed in) and times[6].

Comparison rule (`compare`): every word bit-identical, a NaN matching any NaN. The device evaluates the
transcendentals in fp64 libm (within 1 ulp of exact for exp / log / expm1 / log1p, 2 ulp for pow) before rounding to
fp32, so where the exact value lies within that distance of an fp32 rounding boundary either neighbour is right:
`Libm.near` counts those evaluations and a mismatch is excused only if one happened in the case.
"""
from __future__ import annotations

import contextlib
import math

import mpmath
import numpy as np
import torch

from dpm_solver_b200 import plan as P

PREC = 96                      # working precision of the exact values, bits
ST_S, ST_LAM_S, ST_LAM_0, ST_H, ST_T, ST_NFE, ST_DONE, ST_ACCEPT, ST_ITERS = range(9)
INT_WORDS = (ST_NFE, ST_DONE, ST_ACCEPT, ST_ITERS)
CO_WORDS = 16
LIVE = 11                      # a, c0, c1, c2, w0..w4, alpha_e, sigma_e
ULPS = {"exp": 1, "log": 1, "expm1": 1, "log1p": 1, "pow": 2, "sqrt": 0}    # device error bound, in fp64 ulps


# ---- words ----------------------------------------------------------------------------------------------------------
def f2w(v: float) -> int:
    """fp32 bit pattern of v (rounded to fp32 first)."""
    return int(np.array([v], dtype=np.float32).view(np.uint32)[0])


def w2f(w) -> float:
    return float(np.array([w], dtype=np.uint32).view(np.float32)[0])


def f32(v) -> float:
    return float(np.float32(v))


def compare(got: np.ndarray, want: np.ndarray, float_mask=None) -> list:
    """Indices of words that differ (flat). Words under float_mask (default: all) that are NaN in both match."""
    got, want = np.asarray(got, np.uint32).reshape(-1), np.asarray(want, np.uint32).reshape(-1)
    fm = np.ones(got.shape, bool) if float_mask is None else np.asarray(float_mask, bool).reshape(-1)
    gf, wf = got.view(np.float32), want.view(np.float32)
    same = (got == want) | (fm & np.isnan(gf) & np.isnan(wf))
    return np.nonzero(~same)[0].tolist()


STATE_FLOAT = np.array([i not in INT_WORDS for i in range(16)])


# ---- correctly rounded libm -----------------------------------------------------------------------------------------
def _round32(v, k: int):
    """(fp32 value nearest to the mpf v (ties to even, subnormals, overflow to inf), True if an fp32 rounding
    boundary lies within k fp64 ulps of v)."""
    if mpmath.isnan(v):
        return math.nan, False
    if mpmath.isinf(v):
        return float(v), False
    if v == 0:
        return 0.0, False
    sign = -1.0 if v < 0 else 1.0
    a = abs(v)
    _, e2 = mpmath.frexp(a)                 # a in [2^(e2-1), 2^e2)
    e = int(e2) - 1
    q = max(e, -126) - 23                   # fp32 quantum at a
    y = mpmath.ldexp(a, -q)
    n = int(mpmath.floor(y))
    frac = y - n
    if frac > 0.5 or (frac == 0.5 and n % 2 == 1):
        n += 1
    r = math.ldexp(n, q)
    if r >= 2.0 ** 128:
        r = math.inf
    near = abs(frac - mpmath.mpf(0.5)) * mpmath.ldexp(1, q) <= k * mpmath.ldexp(1, max(e, -1022) - 52)
    return sign * r, bool(near)


class Libm:
    """Correctly rounded fp32 exp / log / expm1 / log1p / sqrt and the reference's float_power; counts the evaluations
    that lie near an fp32 rounding boundary (`near`) and, if `torch_check`, those where torch's own fp32 result
    differs (`torch_differs`, informational)."""

    def __init__(self, torch_check: bool = False):
        self.near = 0
        self.evals = 0
        self.torch_differs = 0
        self.torch_check = torch_check
        self._cache = {}

    def _exact(self, name, x):
        with mpmath.workprec(PREC):
            X = mpmath.mpf(x)
            return {"exp": mpmath.exp, "log": mpmath.log, "expm1": mpmath.expm1, "log1p": mpmath.log1p,
                    "sqrt": mpmath.sqrt}[name](X)

    def unary(self, name: str, x: float) -> float:
        key = (name, x, math.copysign(1.0, x))              # -0.0 == 0.0, but expm1 / log1p keep the sign
        hit = self._cache.get(key)
        if hit is None:
            hit = self._unary(name, x)
            self._cache[key] = hit
        r, near = hit
        self.evals += 1
        self.near += near
        if self.torch_check:
            t = float(_TORCH[name](torch.tensor([x], dtype=torch.float32))[0])
            self.torch_differs += not (t == r or (math.isnan(t) and math.isnan(r)))
        return r

    def _unary(self, name, x):
        # IEEE special values are exact; everything else from the exact value
        if math.isnan(x):
            return math.nan, False
        if name == "exp":
            if math.isinf(x):
                return (math.inf if x > 0 else 0.0), False
        elif name == "log":
            if x < 0:
                return math.nan, False
            if x == 0:
                return -math.inf, False
            if math.isinf(x):
                return math.inf, False
        elif name == "expm1":
            if x == 0:
                return x, False                                   # keeps the sign of zero
            if math.isinf(x):
                return (math.inf if x > 0 else -1.0), False
        elif name == "sqrt":
            if x < 0:
                return math.nan, False
            if x == 0 or math.isinf(x):
                return x, False
        elif name == "log1p":
            if x == 0:
                return x, False
            if x < -1:
                return math.nan, False
            if x == -1:
                return -math.inf, False
            if math.isinf(x):
                return math.inf, False
        with mpmath.workprec(PREC):
            return _round32(self._exact(name, x), ULPS[name])

    def float_power(self, e: float, p: float) -> float:
        """fp32(fp64(e ** p)) for the fp32 e and the python float p < 0 of the reference's float_power(...).float()."""
        self.evals += 1
        if math.isnan(e) or e < 0:
            return math.nan
        if e == 0:
            return math.inf
        if math.isinf(e):
            return 0.0
        with mpmath.workprec(PREC):
            exact = mpmath.power(mpmath.mpf(e), mpmath.mpf(p))
            d = float(exact)                                      # mpmath rounds to nearest double
            r = f32(d)
            _, near = _round32(exact, ULPS["pow"])
        self.near += near
        return r


# ---- the substitution context ---------------------------------------------------------------------------------------
_UNARY = ("exp", "log", "expm1", "log1p", "sqrt")
_NAMES = _UNARY + ("logaddexp", "float_power")
_TORCH = {n: getattr(torch, n) for n in _NAMES}            # the originals, whatever is patched later


def _torch_unary(name):
    fn = _TORCH[name]
    return lambda x: float(fn(torch.tensor([x], dtype=torch.float32))[0])


def _glibc_unary(name):
    """The C library's fp32 function: what ATen's scalar logaddexp kernel calls (std::exp / std::log1p on float),
    where torch.exp / torch.log1p take the vectorised (SLEEF) path even for one element."""
    import ctypes
    import ctypes.util
    fn = getattr(ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6"), name + "f")
    fn.restype, fn.argtypes = ctypes.c_float, [ctypes.c_float]
    return fn


def _std_max(a, b):
    return b if a < b else a                                     # std::max: NaN in `a` survives, in `b` is dropped


@contextlib.contextmanager
def libm(m=None, calls: dict | None = None):
    """Replace torch.exp / log / expm1 / log1p / sqrt / logaddexp / float_power, for the duration, by elementwise versions
    built on `m` (a Libm: correctly rounded), or, if `m` is None, on the functions torch itself evaluates them with
    -- the same plumbing, so `libm(None)` must reproduce the unpatched results bit for bit. `m` False substitutes
    nothing. `calls` (optional) counts the calls per name."""
    if m is False:
        yield
        return
    saved = {n: getattr(torch, n) for n in _NAMES}
    un = {n: (lambda x, n=n: m.unary(n, x)) if m is not None else _torch_unary(n) for n in _UNARY}
    if m is None:       # ATen's scalar logaddexp kernel
        glibc = {n: _glibc_unary(n) for n in ("exp", "log1p")}
        lae = {n: (lambda x, f=f: float(np.float32(f(x)))) for n, f in glibc.items()}
    else:
        lae = un

    def count(n):
        if calls is not None:
            calls[n] = calls.get(n, 0) + 1

    def elementwise(name):
        def f(x, *args, **kw):
            assert not args and not kw and torch.is_tensor(x) and x.dtype == torch.float32, (name, x)
            count(name)
            vals = [un[name](v) for v in x.reshape(-1).tolist()]
            return torch.tensor(vals, dtype=torch.float32).reshape(x.shape)
        return f

    def logaddexp(a, b):
        count("logaddexp")
        a, b = torch.broadcast_tensors(a, b)
        assert a.dtype == b.dtype == torch.float32
        out = []
        for x, y in zip(a.reshape(-1).tolist(), b.reshape(-1).tolist()):
            if math.isinf(x) and x == y:
                out.append(x)
                continue
            mx = np.float32(_std_max(x, y))
            d = float(abs(np.float32(x) - np.float32(y)))
            out.append(float(mx + np.float32(lae["log1p"](lae["exp"](-d)))))
        return torch.tensor(out, dtype=torch.float32).reshape(a.shape)

    def float_power(e, p):
        count("float_power")
        assert torch.is_tensor(e) and e.dtype == torch.float32 and isinstance(p, float)
        if m is None:
            vals = [float(_TORCH["float_power"](torch.tensor(v, dtype=torch.float32), p)) for v in e.reshape(-1).tolist()]
        else:
            vals = [m.float_power(v, p) for v in e.reshape(-1).tolist()]
        return torch.tensor(vals, dtype=torch.float64).reshape(e.shape)

    try:
        for n in _UNARY:
            setattr(torch, n, elementwise(n))
        torch.logaddexp = logaddexp
        torch.float_power = float_power
        yield
    finally:
        for n, f in saved.items():
            setattr(torch, n, f)


# ---- the controller -------------------------------------------------------------------------------------------------
class Cfg:
    """What dpm_adaptive_ctl carries: the schedule (the NoiseScheduleVP the device tables were copied from) and the
    solver options; t_0, theta, t_err are rounded to fp32 as the C struct holds them."""

    def __init__(self, ns, order, algorithm_type, solver_type, t_0, theta=0.9, t_err=1e-5, discrete_input=True):
        self.ns, self.order, self.algo, self.solver_type = ns, order, algorithm_type, solver_type
        self.t_0, self.theta, self.t_err = f32(t_0), f32(theta), f32(t_err)
        self.discrete_input = bool(discrete_input)


def _t(v: float) -> torch.Tensor:
    return torch.tensor([v], dtype=torch.float32)


def _marg(ns, t: torch.Tensor):
    m = P.Marginals(ns, t)
    return float(m.lam), float(m.alpha), float(m.sigma)


def _not_finished(c: Cfg, s: float) -> bool:
    return bool(torch.abs((_t(s) - c.t_0)).mean() > c.t_err)          # while-condition :995


def init(c: Cfg, t_T: float, h_init: float, m: Libm) -> np.ndarray:
    """k_adapt_init (:979-982): s = t_T, lambda_s, lambda_0, h = h_init, the rest 0; done if already at t_0."""
    st = np.zeros(16, np.uint32)
    with libm(m):
        s = _t(f32(t_T))
        lam_s = c.ns.marginal_lambda(s)
        lam_0 = c.ns.marginal_lambda(c.t_0 * torch.ones_like(s))
    st[ST_S], st[ST_LAM_S], st[ST_LAM_0], st[ST_H] = f2w(float(s)), f2w(float(lam_s)), f2w(float(lam_0)), f2w(h_init)
    if not _not_finished(c, float(s)):
        st[ST_DONE] = 1
    return st


def _input_time(c: Cfg, t: float) -> float:
    if not c.discrete_input:
        return t
    return float((_t(t) - 1. / c.ns.total_N) * 1000.)                   # get_model_input_time :278


def _block(co, alsig):
    w = [co.a, co.c0, co.c1, co.c2, co.w0, co.w1, co.w2, co.w3, co.w4, alsig[1], alsig[2]]
    return [f2w(v) for v in w]


def plan(c: Cfg, state: np.ndarray, coef: np.ndarray, times: np.ndarray, m: Libm):
    """k_adapt_plan -> (state, coef, times) after the launch. Live: t = lambda^-1(lambda_s + h) (:996) and the blocks
    of the lower / higher update (:985-992, plan.py); finished: identity blocks and time labels at t_0."""
    st, co, tm = state.copy(), coef.copy(), times.copy()
    ns = c.ns
    with libm(m):
        if st[ST_DONE] != 0:
            m0 = _marg(ns, _t(c.t_0))
            ident = [f2w(v) for v in (1., 0., 0., 0., 1., 1., 1., 1., 1., m0[1], m0[2])]
            for b in range(4):
                co[b, :LIVE] = ident
            tt = [c.t_0] * 3
        else:
            s, lam_s, h = _t(w2f(st[ST_S])), _t(w2f(st[ST_LAM_S])), _t(w2f(st[ST_H]))
            t = ns.inverse_lambda(lam_s + h)
            st[ST_T] = f2w(float(t))
            if c.order == 2:
                low = P.first_update_coeffs(ns, c.algo, s, t)
                high = P.singlestep_second(ns, c.algo, c.solver_type, s, t, 0.5)
                s1 = high.times[1]
                ms, m1 = _marg(ns, s), _marg(ns, s1)
                blocks = [(low, ms), (high.stages[0], ms), (high.stages[1], m1)]
                tt = [float(s), float(s1), float(s)]
            else:
                low = P.singlestep_second(ns, c.algo, c.solver_type, s, t, 1. / 3.)
                high = P.singlestep_third(ns, c.algo, c.solver_type, s, t, 1. / 3., 2. / 3.)
                s1, s2 = high.times[1], high.times[2]
                assert np.array_equal(low.times[1].numpy(), s1.numpy(), equal_nan=True)
                ms, m1, m2 = _marg(ns, s), _marg(ns, s1), _marg(ns, s2)
                blocks = [(low.stages[0], ms), (low.stages[1], m1), (high.stages[1], m1), (high.stages[2], m2)]
                tt = [float(s), float(s1), float(s2)]
            for b, (cf, al) in enumerate(blocks):
                co[b, :LIVE] = _block(cf, al)
        for j in range(3):
            tm[j] = f2w(tt[j])
            tm[3 + j] = f2w(_input_time(c, tt[j]))
    return st, co, tm


def host_update(theta, h, E, order, lambda_0, lambda_s):
    """The host controller's step-size update, solver.py dpm_solver_adaptive (the reference's :1007, verbatim)."""
    return torch.min(theta * h * torch.float_power(E, -1. / order).float(), lambda_0 - lambda_s)


def decide(c: Cfg, state: np.ndarray, E: float, m: Libm | None):
    """k_adapt_decide -> (state, branch). `m` None evaluates float_power with torch's own (for the CPU cross-checks).

    Branches: 'done' (already finished: only accept cleared), 'nan_E' (done = 2: the host raises
    FloatingPointError), 'accept' / 'reject' (:1002-1008), each possibly followed by 'nan_h' (h = NaN, done = 2: every
    later estimate is NaN, the host raises on the next one) and 'finish' (done = 1, |s - t_0| <= t_err)."""
    st = state.copy()
    st[ST_ACCEPT] = 0
    if st[ST_DONE] != 0:
        return st, ["done"]
    st[ST_ITERS] += 1
    E = f32(E)
    if math.isnan(E):
        st[ST_DONE] = 2
        return st, ["nan_E"]
    branch = []
    with libm(m):
        if E <= 1.:
            branch.append("accept")
            st[ST_ACCEPT] = 1
            st[ST_S] = st[ST_T]
            st[ST_LAM_S] = f2w(float(c.ns.marginal_lambda(_t(w2f(st[ST_T])))))
        else:
            branch.append("reject")
        hn = host_update(c.theta, _t(w2f(st[ST_H])), torch.tensor(E, dtype=torch.float32), c.order,
                         _t(w2f(st[ST_LAM_0])), _t(w2f(st[ST_LAM_S])))
    st[ST_H] = f2w(float(hn))
    st[ST_NFE] += c.order
    if float(hn) == f32(w2f(st[ST_LAM_0]) - w2f(st[ST_LAM_S])):
        branch.append("clamp")
    if math.isnan(float(hn)):
        branch.append("nan_h")
        st[ST_DONE] = 2
    if not _not_finished(c, w2f(st[ST_S])):
        branch.append("finish")
        st[ST_DONE] = 1
    return st, branch
