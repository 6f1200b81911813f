"""The oracle of the device step-size controller (tests/adaptive_oracle.py) checked on the CPU before the GPU tests
rely on it: its correctly rounded functions against mpmath, its substitution context against the unpatched
plan.py / schedule.py (with torch's own functions plugged in it must change nothing), its decide() against the host
controller's update, and its linear-schedule lambda^-1 against the reference's, where the device's old form differed."""
import inspect
import math
import random

import mpmath
import numpy as np
import pytest
import torch

import adaptive_oracle as O
from helpers import product_schedule

SCHEDULES = ["sd", "iddpm_cosine", "vp_linear"]


def _nearest_f32(exact):
    """fp32 nearest to the mpf `exact`, by comparing the neighbours of a first guess (independent of _round32)."""
    g = np.float32(float(exact))
    cands = [np.nextafter(g, np.float32(-np.inf)), g, np.nextafter(g, np.float32(np.inf))]
    d = [abs(mpmath.mpf(float(c)) - exact) for c in cands]
    best = min(d)
    ties = [c for c, e in zip(cands, d) if e == best]
    ties.sort(key=lambda c: int(np.array([c], np.float32).view(np.uint32)[0]) & 1)     # ties to the even pattern
    return float(ties[0])


def test_correctly_rounded_functions_match_mpmath():
    rng = random.Random(11)
    m = O.Libm()
    args = {"exp": lambda: rng.uniform(-80, 80), "log": lambda: math.exp(rng.uniform(-80, 80)),
            "sqrt": lambda: math.exp(rng.uniform(-80, 80)),
            "expm1": lambda: rng.choice([1, -1]) * math.exp(rng.uniform(-30, 3.5)),
            "log1p": lambda: rng.choice([math.exp(rng.uniform(-30, 20)), -math.exp(rng.uniform(-30, -1e-3))])}
    n = 0
    with mpmath.workprec(200):
        for name, draw in args.items():
            fn = {"exp": mpmath.exp, "log": mpmath.log, "expm1": mpmath.expm1, "log1p": mpmath.log1p,
                  "sqrt": mpmath.sqrt}[name]
            for _ in range(400):
                x = O.f32(draw())
                assert m.unary(name, x) == _nearest_f32(fn(mpmath.mpf(x))), (name, x)
                if name == "sqrt":
                    assert m.unary(name, x) == float(np.sqrt(np.float32(x)))            # IEEE sqrt
                n += 1
        for e in [1e-45, 1e-40, 1e-30, 0.3, float(np.nextafter(np.float32(1), np.float32(0))), 1.0, 1.0000001, 2.0, 3.4e38]:
            for order in (2, 3):
                e32 = O.f32(e)
                want = O.f32(float(mpmath.power(mpmath.mpf(e32), mpmath.mpf(-1. / order))))
                assert m.float_power(e32, -1. / order) == want, (e, order)
                assert m.float_power(e32, -1. / order) == float(torch.float_power(torch.tensor(e32), -1. / order).float())
                n += 1
    # IEEE specials, and zeros keep their sign
    assert m.unary("exp", -math.inf) == 0.0 and m.unary("exp", math.inf) == math.inf
    assert m.unary("log", 0.0) == -math.inf and math.isnan(m.unary("log", -1.0))
    assert math.copysign(1, m.unary("expm1", -0.0)) == -1 and m.unary("expm1", -math.inf) == -1.0
    assert math.copysign(1, m.unary("log1p", -0.0)) == -1 and m.unary("log1p", -1.0) == -math.inf
    assert m.float_power(0.0, -0.5) == math.inf and m.float_power(math.inf, -0.5) == 0.0
    assert math.isnan(m.float_power(math.nan, -0.5))
    assert m.near == 0 and n >= 2000


def test_boundary_flag_fires_near_a_rounding_boundary():
    one = mpmath.mpf(1)
    with mpmath.workprec(O.PREC):
        mid = one + mpmath.ldexp(1, -24)                       # halfway between 1 and 1 + 2^-23
        assert O._round32(mid, 1) == (1.0, True)               # ties to even
        assert O._round32(mid + mpmath.ldexp(1, -60), 1) == (1.0 + 2 ** -23, True)
        assert O._round32(mid - mpmath.ldexp(1, -53), 1) == (1.0, True)     # within one fp64 ulp
        assert O._round32(mid - mpmath.ldexp(1, -40), 1) == (1.0, False)
        assert O._round32(mpmath.ldexp(3, -150), 1)[0] == 2 ** -148          # subnormal quantum, ties to even
        assert O._round32(mpmath.mpf(2) ** 128, 1)[0] == math.inf
    m = O.Libm()
    x = O.f32(1e-3)
    m._cache[("exp", x, 1.0)] = (O.f32(math.exp(x)), True)     # a result on a boundary is counted as such
    m.unary("exp", x)
    assert m.near == 1


def _states(ns, c):
    """(s, h) over the range the controller sees: h = 0, small, large, beyond lambda_0 - lambda_s, negative."""
    t0 = c.t_0
    out = []
    for s in (1.0, 0.37, 0.05, 3 * t0, t0):
        st = O.init(c, s, 0.05, False)
        D = O.w2f(st[O.ST_LAM_0]) - O.w2f(st[O.ST_LAM_S])
        out += [(s, h) for h in (0.0, 1e-3, 0.2, D, D + 0.5, -0.1)]
    return out


@pytest.mark.parametrize("name", SCHEDULES)
def test_torch_substitution_reproduces_plan_py(name):
    """With torch's own functions plugged into the substitution, init / plan / decide reproduce the unpatched
    plan.py coefficients, schedule.py scalars and host update bit for bit -- the hooks change nothing but the
    functions -- and every hook is reached. Informational: on how many of the oracle's evaluations torch's fp32
    functions differ from the correctly rounded ones."""
    ns = product_schedule(name)
    t0 = 1e-3 if ns.schedule == "linear" else 1. / ns.total_N
    calls = {}
    mcr = O.Libm(torch_check=True)
    n = 0
    for order in (2, 3):
        for algo in ("dpmsolver++", "dpmsolver"):
            for st_type in ("dpmsolver", "taylor"):
                c = O.Cfg(ns, order, algo, st_type, t0, discrete_input=order == 2)
                for s, h in _states(ns, c):
                    co, tm = np.zeros((4, 16), np.uint32), np.zeros(6, np.uint32)
                    res = {}
                    for mode in (False, None):
                        st = O.init(c, s, h, mode)
                        p = O.plan(c, st, co, tm, mode)
                        d = O.decide(c, p[0], 0.7, mode)[0], O.decide(c, p[0], 1.3, mode)[0]
                        res[mode] = (st, *p, *d)
                    for a, b in zip(res[False], res[None]):
                        assert not O.compare(a, b), (order, algo, st_type, s, h)
                    with O.libm(None, calls):                    # (False: plan() adds no context of its own)
                        O.plan(c, res[False][0], co, tm, False)
                    O.plan(c, O.init(c, s, h, mcr), co, tm, mcr)
                    n += 1
    with O.libm(None, calls):
        O.host_update(0.9, torch.ones(1), torch.tensor(0.5), 2, torch.ones(1), torch.zeros(1))
    assert {"exp", "log", "expm1", "sqrt", "logaddexp", "float_power"} <= set(calls), calls
    assert n >= 8 * 30
    print(f"{name}: torch's fp32 exp/log/expm1/sqrt differ from the correctly rounded value on "
          f"{mcr.torch_differs} of {mcr.evals} oracle evaluations ({mcr.near} near a boundary)")


E_GRID = [0.0, 1e-45, 1e-40, float(np.nextafter(np.float32(1), np.float32(0))), 1.0,
          float(np.nextafter(np.float32(1), np.float32(2))), 0.3, 3.4e38, math.inf, math.nan]


def _host_line():
    from dpm_solver_b200.solver import DPM_Solver
    lines = [ln.strip() for ln in inspect.getsource(DPM_Solver.dpm_solver_adaptive).splitlines()
             if ln.strip().startswith("h = torch.min(")]
    assert len(lines) == 1
    return lines[0][len("h = "):]


def test_decide_matches_host_controller_update():
    """decide() (with torch's float_power, and with the correctly rounded one) gives the h of the host controller's
    own update line (solver.py, the reference's :1007 verbatim) on E in {0, denormals, 1 - ulp, 1, 1 + ulp, 0.3,
    3.4e38, inf, NaN} x h in {0, small, normal, clamped by lambda_0 - lambda_s} x order; E = 0 with h = 0 is NaN
    (done = 2), E = inf is 0, a NaN E stops with done = 2 before touching h."""
    expr = _host_line()
    assert expr in inspect.getsource(O.host_update)
    m = O.Libm()
    branches = set()
    n = 0
    for name in ("sd", "vp_linear"):
        ns = product_schedule(name)
        t0 = 1e-3 if ns.schedule == "linear" else 1. / ns.total_N
        for order in (2, 3):
            c = O.Cfg(ns, order, "dpmsolver++", "dpmsolver", t0)
            st = O.init(c, 0.5, 0.05, False)
            st = O.plan(c, st, np.zeros((4, 16), np.uint32), np.zeros(6, np.uint32), False)[0]
            for h in (0.0, 1e-6, 0.05, 30.0):
                st[O.ST_H] = O.f2w(h)
                for E in E_GRID:
                    got, br = O.decide(c, st, E, None)
                    got_cr, _ = O.decide(c, st, E, m)
                    branches.update(br)
                    n += 1
                    if math.isnan(E):
                        assert br == ["nan_E"] and got[O.ST_DONE] == 2 and got[O.ST_H] == st[O.ST_H]
                        continue
                    lam_s = O.w2f(got[O.ST_LAM_S])
                    want = eval(expr, {"torch": torch}, dict(
                        theta=0.9, h=torch.tensor([h], dtype=torch.float32), E=torch.tensor(O.f32(E)), order=order,
                        lambda_0=torch.tensor([O.w2f(st[O.ST_LAM_0])]), lambda_s=torch.tensor([lam_s])))
                    assert not O.compare([got[O.ST_H]], [O.f2w(float(want))]), (name, order, h, E)
                    assert not O.compare(got_cr, got, O.STATE_FLOAT), (name, order, h, E)
                    if E == 0.0 and h == 0.0:
                        assert math.isnan(O.w2f(got[O.ST_H])) and got[O.ST_DONE] == 2
                    if E == math.inf:
                        assert O.w2f(got[O.ST_H]) == 0.0
    assert {"nan_E", "accept", "reject", "clamp", "nan_h"} <= branches and n == 2 * 2 * 4 * len(E_GRID)


def test_linear_inverse_lambda_matches_reference_where_device_form_differed():
    """schedule.py's linear lambda^-1 squares beta_0 in double, as the reference does (:162); the device used to
    square fl32(beta_0) and so differs from it on thousands of lambda in [3.3, 11.4] -- t in (1e-9, 7.5e-3), where
    every solve on 'linear' ends. There the oracle (schedule.py, correctly rounded functions) equals the reference's
    own inverse_lambda under the same functions, and the fl32(beta_0) square does not."""
    from oracle import ref_loader
    ns = product_schedule("vp_linear")
    b0, b1 = ns.beta_0, ns.beta_1
    lam = torch.from_numpy(np.linspace(-12, 12, 200001).astype(np.float32))

    def device_form(lamb):
        tmp = 2. * (b1 - b0) * torch.logaddexp(-2. * lamb, torch.zeros((1,)).to(lamb))
        b = torch.tensor(b0, dtype=torch.float32)
        return tmp / (torch.sqrt(b * b + tmp) + b0) / (b1 - b0)

    a, d = ns.inverse_lambda(lam), device_form(lam)
    diff = lam[a != d]
    assert diff.numel() > 10000 and float(diff.min()) >= 3.3 and float(diff.max()) <= 11.4, \
        (diff.numel(), float(diff.min()), float(diff.max()))
    ref = ref_loader.load("dpm_solver_pytorch").NoiseScheduleVP("linear", continuous_beta_0=b0, continuous_beta_1=b1) \
        if ref_loader.available() else None

    def literal(lamb):                                      # the reference's :161-163
        tmp = 2. * (b1 - b0) * torch.logaddexp(-2. * lamb, torch.zeros((1,)).to(lamb))
        Delta = b0 ** 2 + tmp
        return tmp / (torch.sqrt(Delta) + b0) / (b1 - b0)

    m = O.Libm()
    sample = diff[torch.randperm(diff.numel(), generator=torch.Generator().manual_seed(3))[:300]]
    still = 0
    with O.libm(m):
        for v in sample.tolist():
            x = torch.tensor([v], dtype=torch.float32)
            want = ns.inverse_lambda(x)
            assert torch.equal(want, literal(x)), v
            if ref is not None:
                assert torch.equal(want, ref.inverse_lambda(x)), v
            still += not torch.equal(want, device_form(x))
    assert still >= 100 and m.near == 0, still
