"""T4: properties that do not depend on the reference at all (run on the numpy executor).

For Gaussian data x0 ~ N(0, s^2 I) the optimal noise predictor is closed form,
eps*(x,t) = sigma_t x / (alpha_t^2 s^2 + sigma_t^2), the diffusion ODE is linear and its exact
solution is x_t = x_T * sqrt((alpha_t^2 s^2 + sigma_t^2) / (alpha_T^2 s^2 + sigma_T^2)).
The global error of an order-p solver must fall like h^p."""
import math

import numpy as np
import pytest
import torch


def exact_setup(s=0.7):
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper
    ns = NoiseScheduleVP("linear", continuous_beta_0=0.1, continuous_beta_1=20.)

    def net(x, t):
        al = ns.marginal_alpha(t).reshape(-1, 1, 1, 1).double()
        sg = ns.marginal_std(t).reshape(-1, 1, 1, 1).double()
        return (sg * x.double() / (al * al * s * s + sg * sg)).float()

    def truth(x_T, t_T, t_0):
        v = lambda t: float(ns.marginal_alpha(torch.tensor([t])).double() ** 2 * s * s + ns.marginal_std(torch.tensor([t])).double() ** 2)
        return x_T.double() * math.sqrt(v(t_0) / v(t_T))

    return ns, model_wrapper(net, ns), truth


@pytest.mark.parametrize("algo", ["dpmsolver++", "dpmsolver"])
# multistep-3 starts with one order-1 and one order-2 step (sample() :1185-1193): their O(h^2) local error
# bounds the observed global order between 2 and 3
@pytest.mark.parametrize("method,order,expected", [("multistep", 1, 1), ("multistep", 2, 2), ("multistep", 3, 2.3),
                                                   ("singlestep_fixed", 2, 2), ("singlestep_fixed", 3, 3)])
def test_empirical_convergence_order(oracle_backend, algo, method, order, expected):
    from dpm_solver_b200 import DPM_Solver
    ns, fn, truth = exact_setup()
    x_T = torch.randn(2, 3, 8, 8, generator=torch.Generator().manual_seed(0))
    t_T, t_0 = 0.8, 0.1                       # moderate logSNR span keeps fp32 noise below the truncation error
    ref = truth(x_T, t_T, t_0)
    errs = []
    grid = (12, 24, 48) if order < 3 else (12, 24)
    for n in grid:
        s = DPM_Solver(fn, ns, algorithm_type=algo)
        y = s.sample(x_T, steps=n * (order if method != "multistep" else 1), t_start=t_T, t_end=t_0, order=order,
                     skip_type="logSNR", method=method, lower_order_final=False)
        errs.append(float((y.double() - ref).abs().max()))
    slopes = [math.log2(errs[i] / errs[i + 1]) for i in range(len(errs) - 1)]
    assert all(e > 0 for e in errs)
    assert min(slopes) > expected - 0.45, (errs, slopes)


def test_more_steps_converge_to_truth(oracle_backend):
    from dpm_solver_b200 import DPM_Solver
    ns, fn, truth = exact_setup()
    x_T = torch.randn(2, 3, 8, 8, generator=torch.Generator().manual_seed(1))
    y = DPM_Solver(fn, ns).sample(x_T, steps=60, t_start=1.0, t_end=1e-3, order=3, skip_type="logSNR")
    ref = truth(x_T, 1.0, 1e-3)
    assert float((y.double() - ref).abs().max() / ref.abs().max()) < 2e-3   # fp32 schedule scalars bound the floor


def test_sample_then_inverse_round_trip(oracle_backend):
    from dpm_solver_b200 import DPM_Solver
    ns, fn, _ = exact_setup()
    x = torch.randn(2, 3, 8, 8, generator=torch.Generator().manual_seed(2))
    s = DPM_Solver(fn, ns)
    y = s.sample(x, steps=40, t_start=0.9, t_end=0.05, order=3, skip_type="logSNR")
    xr = s.inverse(y, steps=40, t_start=0.05, t_end=0.9, order=3, skip_type="logSNR")
    assert float((xr - x).abs().max() / x.abs().max()) < 1e-3


# ---- the kernels' constant division (csrc/common.cuh: div_const) in exact rational arithmetic ----------------
def _rn32(fr):
    """Round a Fraction to the nearest float32 (ties to even), exactly."""
    from fractions import Fraction
    if fr == 0:
        return np.float32(0.0)
    c = np.float32(float(fr))                       # within one ulp of the answer (double rounding at worst)
    cands = {float(c), float(np.nextafter(c, np.float32(np.inf))), float(np.nextafter(c, np.float32(-np.inf)))}
    best = None
    for v in cands:
        err = abs(Fraction(v) - fr)
        even = (np.float32(v).view(np.uint32) & 1) == 0
        key = (err, 0 if even else 1)
        if best is None or key < best[0]:
            best = (key, v)
    return np.float32(best[1])


def test_two_step_constant_division_is_correctly_rounded():
    """q0 = RN(x*r), then twice: e = x - q*d (one FMA), q = RN(q + e*r), with r = RN(1/d): equals RN(x/d) for every
    divisor the kernels accept (recip_div_ok: |d| in [2^-20, 2^21), biased exponent 107..147, significand not all
    ones). After the first refinement the quotient is faithful, so the second residual is EXACT (asserted) -- the
    premise of Markstein's theorem. Random and adversarial pairs over the whole admitted range: every exponent,
    quotients next to rounding midpoints, divisors one ulp from a power of two or from the excluded all-ones pattern,
    numerators within a few ulps of the range guard (1e-25, 1e30), there too with quotients next to a midpoint."""
    from fractions import Fraction
    from step_edges import from_bits, nudge, recip_div_ok
    rng = np.random.default_rng(7)
    ds = []
    for _ in range(300):
        ds.append(np.float32(rng.uniform(0.5, 2.0) * 2.0 ** rng.integers(-19, 19)))
    for e in (-19, -3, 0, 1, 7, 18):
        base = np.float32(2.0 ** e)
        ds += [base, np.nextafter(base, np.float32(np.inf)), np.nextafter(np.nextafter(base, np.float32(0)), np.float32(0))]
    for e in range(-20, 21):                          # biased exponents 107..147
        all_ones = from_bits(((e + 127) << 23) | 0x7fffff)
        ds += [np.float32(rng.uniform(1.0, 2.0) * 2.0 ** e), nudge(all_ones, -1), nudge(all_ones, 1),
               from_bits((e + 127) << 23)]
    checked = 0
    for d in ds:
        if not recip_div_ok(d):
            continue                                  # refused on the host (IEEE path)
        d = np.float32(d)
        r = np.float32(1.0) / d                       # numpy's fp32 division is correctly rounded
        assert _rn32(Fraction(1) / Fraction(float(d))) == r
        xs = [np.float32(rng.standard_normal() * 10.0 ** rng.integers(-6, 6)) for _ in range(12)]
        for _ in range(12):                           # quotients right at / next to a rounding midpoint
            q = np.float32(rng.uniform(1.0, 2.0) * 2.0 ** rng.integers(-10, 10))
            mid = (Fraction(float(q)) + Fraction(float(np.nextafter(q, np.float32(np.inf))))) / 2
            x0 = _rn32(mid * Fraction(float(d)))
            xs += [x0, np.nextafter(x0, np.float32(np.inf)), np.nextafter(x0, np.float32(-np.inf))]
        for g in (1e-25, 1e30):                       # at the guard: x a few ulps from it, and midpoint quotients
            xs += [nudge(g, k) for k in range(-3, 4)]
            q = _rn32(Fraction(float(np.float32(g))) / Fraction(float(d)))
            for k in (-1, 0, 1):
                qk = nudge(q, k)
                mid = (Fraction(float(qk)) + Fraction(float(np.nextafter(qk, np.float32(np.inf))))) / 2
                x0 = _rn32(mid * Fraction(float(d)))
                xs += [x0, nudge(x0, 1), nudge(x0, -1)]
        for x in xs:
            x = np.float32(x) * np.float32(rng.choice([-1.0, 1.0]))
            if not (1e-25 < abs(float(x)) < 1e30):
                continue
            fx, fd, fr_ = Fraction(float(x)), Fraction(float(d)), Fraction(float(r))
            q = _rn32(fx * fr_)
            e = _rn32(fx - Fraction(float(q)) * fd)
            q = _rn32(Fraction(float(q)) + Fraction(float(e)) * fr_)
            e = _rn32(fx - Fraction(float(q)) * fd)
            assert Fraction(float(e)) == fx - Fraction(float(q)) * fd, "the residual of a faithful quotient is exact"
            q = _rn32(Fraction(float(q)) + Fraction(float(e)) * fr_)
            assert q == _rn32(fx / fd), (float(x), float(d))
            checked += 1
    assert checked > 10000
