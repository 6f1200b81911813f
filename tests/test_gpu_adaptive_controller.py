"""The step-size controller of dpm_solver_adaptive on the device (csrc/adaptive_ctl.cu: k_adapt_init, k_adapt_plan,
k_adapt_decide), driven directly through ops.AdaptiveController -- write the state and E, launch, read back -- and
compared word for word with tests/adaptive_oracle.py: the reference's fp32 arithmetic with correctly rounded
exp / log / expm1 / log1p / sqrt and the reference's float_power. Every word the kernels write must be bit-identical (NaN
matches NaN); a mismatch is excused only where the oracle met an fp32 rounding boundary within the device fp64 libm's
error (counted and printed; none are expected), and no test passes without reaching a floor of cases and every
schedule kind, algorithm, order, solver type and controller branch it covers."""
import math
import random

import numpy as np
import pytest
import torch

import adaptive_oracle as O
from helpers import product_schedule

SCHEDULES = ["sd", "ddpm_linear", "iddpm_cosine", "short9", "vp_linear", "linear_b05_15"]
ALGOS = ["dpmsolver++", "dpmsolver"]
TYPES = ["dpmsolver", "taylor"]
SENT = O.f2w(-1234.5)                # coefficient / time words the kernel must not touch
_NS = {}


def schedule(name):
    if name not in _NS:
        from dpm_solver_b200 import NoiseScheduleVP
        if name == "linear_b05_15":
            _NS[name] = NoiseScheduleVP("linear", continuous_beta_0=0.05, continuous_beta_1=15.)
        elif name == "short9":      # a 9-entry table whose knot 5 is on the tie rule: lambda and sigma change with it
            rng = np.random.default_rng(2)
            ac = np.cumprod(1 - np.linspace(1e-3, 0.05, 9) * (1 + 0.3 * rng.random(9)))
            _NS[name] = NoiseScheduleVP("discrete", alphas_cumprod=torch.from_numpy(ac))
        else:
            _NS[name] = product_schedule(name)
    return _NS[name]


def t0_of(ns):
    return 1e-3 if ns.schedule == "linear" else 1. / ns.total_N


def _put(t, words):
    t.view(torch.int32).copy_(torch.from_numpy(np.asarray(words, np.uint32).view(np.int32).reshape(t.shape)))


def _get(t):
    return t.view(torch.int32).cpu().numpy().view(np.uint32).copy()


class Rig:
    """One AdaptiveController and the oracle configuration it mirrors."""

    def __init__(self, be, name, order, algo, solver_type, discrete_input, theta=0.9, t_err=1e-5):
        ns = schedule(name)
        self.name, self.ns = name, ns
        self.kind = ns.schedule
        self.cfg = O.Cfg(ns, order, algo, solver_type, t0_of(ns), theta, t_err, discrete_input)
        self.ctl = be.adaptive_controller(ns, torch.device("cuda:0"), order=order, predict_x0=algo == "dpmsolver++",
                                          taylor=solver_type == "taylor", t_0=t0_of(ns), theta=theta, t_err=t_err,
                                          discrete_input=discrete_input)
        self.key = (self.kind, algo, solver_type, order, bool(discrete_input))

    def init(self, t_T, h):
        self.ctl.init(t_T, h)
        return _get(self.ctl.state)

    def plan(self, state, coef, times):
        _put(self.ctl.state, state)
        _put(self.ctl.coef, coef)
        _put(self.ctl.times, times)
        self.ctl.plan()
        return _get(self.ctl.state), _get(self.ctl.coef), _get(self.ctl.times)

    def decide(self, state, E):
        _put(self.ctl.state, state)
        _put(self.ctl.E, [O.f2w(E)])
        self.ctl.decide()
        return _get(self.ctl.state)


class Tally:
    """Cases run, boundary cases excused, and what the cases reached."""

    def __init__(self, m):
        self.m, self.cases, self.boundary, self.seen = m, 0, [], set()

    def check(self, what, near_before, pairs, ctx):
        """pairs: (got, want, float_mask) word arrays of one case. Fails on a mismatch unless the oracle met a
        rounding boundary while computing this case."""
        self.cases += 1
        bad = {name: O.compare(g, w, fm) for name, (g, w, fm) in pairs.items()}
        bad = {k: v for k, v in bad.items() if v}
        if not bad:
            return True
        if self.m.near > near_before:
            self.boundary.append((what, ctx, bad))
            print("boundary case", what, ctx, bad)
            return False
        detail = {k: [(i, hex(int(pairs[k][0].reshape(-1)[i])), hex(int(pairs[k][1].reshape(-1)[i])),
                       O.w2f(pairs[k][0].reshape(-1)[i]), O.w2f(pairs[k][1].reshape(-1)[i])) for i in v[:6]]
                  for k, v in bad.items()}
        raise AssertionError(f"{what} {ctx}: words differ (index, got, want): {detail}")

    def report(self, name):
        print(f"{name}: {self.cases} cases, {len(self.boundary)} boundary cases, {self.m.evals} correctly rounded "
              f"evaluations ({self.m.near} near a boundary)")


def _fresh_out():
    return np.full((4, 16), SENT, np.uint32), np.full(6, SENT, np.uint32)


def _plan_pairs(dev, ora):
    return {"state": (dev[0], ora[0], O.STATE_FLOAT), "coef": (dev[1], ora[1], None), "times": (dev[2], ora[2], None)}


def _tie_knots(x, y):
    """Knots x[k] at which the reference's bracket (x at a knot takes the interval on its left) and the interval on
    its right interpolate to different fp32 values: the only places where the tie rule is observable."""
    out = []
    for k in range(1, len(x) - 1):
        left = y[k - 1] + (x[k] - x[k - 1]) * (y[k] - y[k - 1]) / (x[k] - x[k - 1])
        right = y[k] + (x[k] - x[k]) * (y[k + 1] - y[k]) / (x[k + 1] - x[k])
        if left != right:
            out.append(float(x[k]))
    return out


def _s_grid(ns, t0):
    if ns.schedule == "discrete":
        ta = ns.t_array.reshape(-1)
        K = ta.numel()
        knots = [float(ta[k]) for k in (K - 1, K // 2, 37, 1, 0) if k < K]
        between = [float((ta[k] + ta[k + 1]) / 2) for k in (K // 3, 5) if k + 1 < K]
        grid = knots + between + _tie_knots(ta.numpy(), ns.log_alpha_array.reshape(-1).numpy())
    else:
        grid = [1.0, 0.5, 0.0371, 0.0123, 2e-3]
    near = [float(np.nextafter(np.float32(t0), np.float32(1)) + np.float32(3e-7)), t0 * 1.5, t0]
    return grid + near


def _h_grid(D):
    return [0.0, 1e-4, 1e-3, 0.01, 0.05, 0.3, 1.0, 3.0, D, D + 0.05, D + 1.0, -0.01, -0.3]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCHEDULES)
def test_plan_matches_oracle(cuda_backend, name):
    """k_adapt_init + k_adapt_plan at s on the table knots, between them, at 1 and near t_0, with h from 0 and 1e-4
    up to lambda_0 - lambda_s and beyond (t, s1, s2 extrapolated below t_0) and negative (above 1): ST_T, the four
    coefficient blocks (the words a launch does not own included) and the six time labels, bitwise; a state within
    t_err of t_0 takes the finished branch (identity blocks at t_0)."""
    m = O.Libm()
    tally = Tally(m)
    seen = set()
    for order in (2, 3):
        for algo in ALGOS:
            for st_type in TYPES:
                rigs = [Rig(cuda_backend, name, order, algo, st_type, di) for di in (True, False)]
                k = 0
                for s in _s_grid(rigs[0].ns, rigs[0].cfg.t_0):
                    st0 = O.init(rigs[0].cfg, s, 0.05, m)
                    D = O.w2f(st0[O.ST_LAM_0]) - O.w2f(st0[O.ST_LAM_S])
                    for hv in _h_grid(D):
                        rig = rigs[k % 2]
                        k += 1
                        near0 = m.near
                        want0 = O.init(rig.cfg, s, hv, m)
                        got0 = rig.init(s, hv)
                        co, tm = _fresh_out()
                        ora = O.plan(rig.cfg, want0, co, tm, m)
                        dev = rig.plan(got0, co, tm)
                        if tally.check("init", near0, {"state": (got0, want0, O.STATE_FLOAT)}, (rig.key, s, hv)):
                            tally.check("plan", near0, _plan_pairs(dev, ora), (rig.key, s, hv))
                        seen.add(rig.key)
                        if want0[O.ST_DONE]:
                            seen.add("done")
                        else:
                            seen.update({"h0"} if hv == 0.0 else {"beyond"} if hv > D else {"neg"} if hv < 0 else set())
    tally.report(f"plan[{name}]")
    assert tally.cases >= 8 * 8 * 13 * 2                 # configurations x s x h x (init, plan)
    kind = schedule(name).schedule
    assert {(kind, a, t, o, d) for a in ALGOS for t in TYPES for o in (2, 3) for d in (True, False)} <= seen
    assert {"done", "h0", "beyond", "neg"} <= seen
    if name == "short9":
        assert _tie_knots(schedule(name).t_array.reshape(-1).numpy(), schedule(name).log_alpha_array.reshape(-1).numpy())


def _boundary_ts(t0, t_err):
    """fp32 t_T around the two edges of |t_T - t_0| <= t_err, three ulps either side."""
    out = []
    for edge in (np.float32(t0) + np.float32(t_err), np.float32(t0) - np.float32(t_err)):
        v = np.float32(edge)
        for _ in range(3):
            v = np.nextafter(v, np.float32(-1))
        for _ in range(7):
            out.append(float(v))
            v = np.nextafter(v, np.float32(2))
    return out


@pytest.mark.gpu
def test_init_matches_oracle(cuda_backend):
    """k_adapt_init: s, lambda_s, lambda_0, h and the zeroed words bitwise; the done flag at t_T = t_0 +- t_err and
    three ulps either side, where it must switch on both edges."""
    m = O.Libm()
    tally = Tally(m)
    flips = 0
    for name in SCHEDULES:
        rig = Rig(cuda_backend, name, 2, "dpmsolver++", "dpmsolver", True)
        t0 = rig.cfg.t_0
        edges = _boundary_ts(t0, rig.cfg.t_err)
        for i, t_T in enumerate([1.0, 0.7, 0.2, t0] + edges):
            for h in (0.05, 0.0, 1.7):
                near0 = m.near
                want = O.init(rig.cfg, t_T, h, m)
                got = rig.init(t_T, h)
                tally.check("init", near0, {"state": (got, want, O.STATE_FLOAT)}, (name, t_T, h))
        dones = [int(O.init(rig.cfg, t, 0.05, m)[O.ST_DONE]) for t in edges]
        flips += (dones[:7] != sorted(dones[:7], reverse=True)) + (dones[7:] != sorted(dones[7:]))   # one switch per edge
        assert 0 in dones[:7] and 1 in dones[:7] and 0 in dones[7:] and 1 in dones[7:], (name, dones)
    tally.report("init")
    assert flips == 0
    assert tally.cases >= len(SCHEDULES) * 18 * 3


E_GRID = [0.0, 1e-45, 1e-40, float(np.nextafter(np.float32(1), np.float32(0))), 1.0,
          float(np.nextafter(np.float32(1), np.float32(2))), 0.3, 2.0, 3.4e38, math.inf, math.nan]


@pytest.mark.gpu
@pytest.mark.parametrize("order", [2, 3])
def test_decide_matches_oracle(cuda_backend, order):
    """k_adapt_decide on E in {0, denormals, 1 - ulp, 1, 1 + ulp, 0.3, 2, 3.4e38, inf, NaN} x h in {0, small, normal,
    lambda_0 - lambda_s and beyond}: all 16 state words. E = 0 with h = 0 is h = NaN (torch.min keeps it: done = 2),
    E = inf is h = 0, a NaN E is done = 2; an accepted step onto t_0 finishes, a finished state only clears accept."""
    m = O.Libm()
    tally = Tally(m)
    branches = set()
    for name in ("sd", "vp_linear", "linear_b05_15"):
        rig = Rig(cuda_backend, name, order, "dpmsolver++", "dpmsolver", True)
        t0 = rig.cfg.t_0
        for s, t_next in [(0.6, None), (0.01, None), (2 * t0, t0), (2 * t0, t0 + 2e-6)]:
            base = O.init(rig.cfg, s, 0.05, m)
            co, tm = _fresh_out()
            base = O.plan(rig.cfg, base, co, tm, m)[0]
            if t_next is not None:
                base[O.ST_T] = O.f2w(t_next)
            D = O.w2f(base[O.ST_LAM_0]) - O.w2f(base[O.ST_LAM_S])
            for h in (0.0, 1e-6, 0.05, D, D + 1.0):
                for E in E_GRID:
                    for done in (0, 1, 2):
                        if done and E not in (0.5, 1.0):
                            continue
                        st = base.copy()
                        st[O.ST_H], st[O.ST_DONE] = O.f2w(h), done
                        st[O.ST_NFE], st[O.ST_ITERS], st[O.ST_ACCEPT] = 6, 3, 1
                        near0 = m.near
                        want, br = O.decide(rig.cfg, st, E, m)
                        got = rig.decide(st, E)
                        tally.check("decide", near0, {"state": (got, want, O.STATE_FLOAT)}, (name, s, t_next, h, E, done))
                        branches.update(br)
                        if E == 0.0 and h == 0.0 and not done and t_next is None:
                            assert math.isnan(O.w2f(got[O.ST_H])) and got[O.ST_DONE] == 2, got
                        if E == math.inf and h > 0 and not done:
                            assert O.w2f(got[O.ST_H]) == 0.0, got
    tally.report(f"decide[order {order}]")
    assert tally.cases >= 3 * 4 * 5 * (len(E_GRID) + 2)
    assert {"done", "nan_E", "accept", "reject", "clamp", "nan_h", "finish"} <= branches, branches


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCHEDULES)
def test_trajectories_match_oracle(cuda_backend, name):
    """plan -> synthetic E -> decide, iterated from t_T = 1 until done and `adaptive_chunk` iterations beyond, for
    both algorithms, solver types and orders: seeded E sequences with rejections; state, blocks and time labels
    compared after every launch."""
    from dpm_solver_b200 import DPM_Solver
    m = O.Libm()
    tally = Tally(m)
    seen, iters, acc, rej = set(), 0, 0, 0
    for i, (order, algo, st_type) in enumerate([(o, a, t) for o in (2, 3) for a in ALGOS for t in TYPES]):
        rig = Rig(cuda_backend, name, order, algo, st_type, i % 2 == 0)
        rng = random.Random(f"{name}/{order}/{algo}/{st_type}")
        want = O.init(rig.cfg, 1.0, 0.05, m)
        got = rig.init(1.0, 0.05)
        co, tm = _fresh_out()
        extra = None
        for it in range(400):
            near0 = m.near
            ora = O.plan(rig.cfg, want, co, tm, m)
            dev = rig.plan(got, co, tm)
            if not tally.check("plan", near0, _plan_pairs(dev, ora), (rig.key, it)):
                break
            co, tm = ora[1], ora[2]
            E = rng.choice([1.0, 0.0]) if rng.random() < 0.04 else float(np.float32(math.exp(rng.gauss(-0.6, 0.9))))
            want, br = O.decide(rig.cfg, ora[0], E, m)
            got = rig.decide(dev[0], E)
            if not tally.check("decide", near0, {"state": (got, want, O.STATE_FLOAT)}, (rig.key, it, E)):
                break
            iters += 1
            acc += "accept" in br
            rej += "reject" in br
            if want[O.ST_DONE] and extra is None:
                extra = DPM_Solver.adaptive_chunk
            if extra is not None:
                extra -= 1
                if extra < 0:
                    break
        assert want[O.ST_DONE] == 1, (rig.key, O.w2f(want[O.ST_S]))
        seen.add(rig.key[:4])
    tally.report(f"trajectories[{name}]")
    kind = schedule(name).schedule
    assert {(kind, a, t, o) for a in ALGOS for t in TYPES for o in (2, 3)} <= seen
    assert iters >= 8 * 10 and acc >= 8 * 5 and rej >= 8
