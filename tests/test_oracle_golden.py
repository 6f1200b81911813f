"""Pin the oracle (oracle/dpm_oracle.py) against golden outputs of the unmodified reference.

numpy namespace: independent arithmetic -- exp/log/expm1 may differ from torch by an ulp, so the
tolerance is a few fp32 ulps on scalars and 2e-6 relative on tensors; where no transcendental is
involved (interpolation, linspace, quantile, element-wise forms) it must be bit-exact.
torch-CPU namespace (the one bench.py times as the CPU baseline): bit-exact everywhere."""
import numpy as np
import pytest
import torch

from cases import SAMPLE_CASES, SCHEDULES, make_betas
from helpers import CASES, oracle_schedule, rel_err, run_oracle_case
from oracle import dpm_oracle as O

TH = O.torch_namespace()


@pytest.mark.parametrize("name", SCHEDULES)
def test_schedule_scalars(golden, name):
    g = golden["schedules"]
    ns = oracle_schedule(name)
    if ns.schedule == "discrete":
        np.testing.assert_array_equal(ns.t, g[f"{name}/t_array"])               # linspace emulation is exact
        np.testing.assert_allclose(ns.log_alpha, g[f"{name}/log_alpha_array"], rtol=3e-7, atol=1e-9)
        assert ns.total_N == int(g[f"{name}/total_N"])
        ns.set_tables(g[f"{name}/t_array"], g[f"{name}/log_alpha_array"])
        np.testing.assert_array_equal(ns.marginal_log_mean_coeff(g[f"{name}/q"]), g[f"{name}/log_alpha"])  # no transcendental
    q = g[f"{name}/q"]
    np.testing.assert_allclose(ns.marginal_log_mean_coeff(q), g[f"{name}/log_alpha"], rtol=1e-6)
    np.testing.assert_allclose(ns.marginal_alpha(q), g[f"{name}/alpha"], rtol=3e-7)
    # operating range of the solver is [1/N, T]; below it 1 - exp(2 log alpha) keeps only a few bits
    fin = np.isfinite(g[f"{name}/lambda"]) & (q >= 9e-4)
    # sigma = sqrt(1 - exp(2 log alpha)) cancels catastrophically as t -> 0 (log alpha ~ -1e-5): one
    # ulp of numpy's exp() vs torch's moves sigma by ~1e-5 absolute and lambda = log alpha - log sigma
    # by ~2e-3 there. (The torch-namespace test below is bit-exact on the same points.)
    np.testing.assert_allclose(ns.marginal_std(q)[fin], g[f"{name}/sigma"][fin], rtol=2e-4, atol=1e-5)
    np.testing.assert_allclose(ns.marginal_lambda(q)[fin], g[f"{name}/lambda"][fin], rtol=2e-4, atol=3e-3)
    np.testing.assert_allclose(ns.inverse_lambda(g[f"{name}/lq"]), g[f"{name}/inv_lambda"], rtol=2e-5, atol=1e-6)


@pytest.mark.parametrize("name", SCHEDULES)
def test_schedule_scalars_torch_namespace_bit_exact(golden, name):
    g = golden["schedules"]
    ns = oracle_schedule(name, xp=TH)
    q = torch.from_numpy(g[f"{name}/q"])
    if ns.schedule == "discrete":
        assert torch.equal(ns.log_alpha, torch.from_numpy(g[f"{name}/log_alpha_array"]))
    for fn, key in ((ns.marginal_log_mean_coeff, "log_alpha"), (ns.marginal_alpha, "alpha"), (ns.marginal_std, "sigma"),
                    (ns.marginal_lambda, "lambda")):
        np.testing.assert_array_equal(fn(q).numpy(), g[f"{name}/{key}"])
    np.testing.assert_array_equal(ns.inverse_lambda(torch.from_numpy(g[f"{name}/lq"])).numpy(), g[f"{name}/inv_lambda"])


@pytest.mark.parametrize("name", SCHEDULES)
def test_time_grids_and_orders(golden, name):
    g = golden["schedules"]
    ns = oracle_schedule(name, g)
    t0 = 1. / ns.total_N
    for N in (5, 15, 20, 50):
        np.testing.assert_array_equal(O.time_steps(ns, "time_uniform", ns.T, t0, N), g[f"{name}/grid/time_uniform/{N}"])
        np.testing.assert_array_equal(O.time_steps(ns, "time_quadratic", ns.T, t0, N), g[f"{name}/grid/time_quadratic/{N}"])
        np.testing.assert_allclose(O.time_steps(ns, "logSNR", ns.T, t0, N), g[f"{name}/grid/logSNR/{N}"], rtol=3e-4, atol=1e-6)
    for steps in (6, 7, 8, 15, 20):
        for order in (1, 2, 3):
            assert O.singlestep_orders(steps, order) == g[f"{name}/ss/time_uniform/{steps}/{order}/orders"].tolist()


def _update_cases(g, ns, algo, xp, conv):
    x, m0, m1, m2 = (conv(g[k]) for k in ("x", "m0", "m1", "m2"))
    ts = xp.linspace(ns.T, 1. / ns.total_N, 21)
    net = lambda xx, tt: 0.3 * xx - 0.1
    # DPM_Solver.model_fn: the network predicts noise; dpmsolver++ buffers x0 (:444-451)
    lin = (lambda xx, tt: O.data_prediction(ns, xx, net(xx, tt), tt)) if algo == "dpmsolver++" else net
    for i in (3, 10, 19):
        T = lambda j: ts[j:j + 1]
        yield f"{i}/first", O.first_update(ns, algo, x, T(i - 1), T(i), m0)
        for st in ("dpmsolver", "taylor"):
            yield f"{i}/ms2/{st}", O.multistep_second(ns, algo, st, x, [m1, m0], [T(i - 2), T(i - 1)], T(i))
            yield f"{i}/ms3/{st}", O.multistep_third(ns, algo, x, [m2, m1, m0], [T(i - 3), T(i - 2), T(i - 1)], T(i))
            yield f"{i}/ss2/{st}", O.singlestep_second(ns, algo, st, x, T(i - 1), T(i), lin)[0]
            yield f"{i}/ss3/{st}", O.singlestep_third(ns, algo, st, x, T(i - 1), T(i), lin)[0]


@pytest.mark.parametrize("sname", ["sd", "vp_linear"])
@pytest.mark.parametrize("algo", ["dpmsolver++", "dpmsolver"])
def test_updates(golden, sname, algo):
    g = golden["updates"]
    ns = oracle_schedule(sname, golden["schedules"])
    for key, got in _update_cases(g, ns, algo, O.NP, lambda a: a):
        assert rel_err(got, g[f"{sname}/{algo}/{key}"]) < 2e-5, key   # numpy expm1 ulp x phi_3 cancellation (SURVEY hard part 1)
    ns = oracle_schedule(sname, xp=TH)
    for key, got in _update_cases(g, ns, algo, TH, torch.from_numpy):
        np.testing.assert_array_equal(got.numpy(), g[f"{sname}/{algo}/{key}"], err_msg=key)


def test_glue(golden):
    g = golden["glue"]
    ns = oracle_schedule("sd", golden["schedules"])
    x, bank, t = g["x"], g["bank"], g["t"]
    B = x.shape[0]
    for mt in ("noise", "x_start", "v", "score"):
        assert rel_err(O.to_noise(ns, mt, x, bank[:B], t), g[f"param/{mt}"]) < 1e-6
    np.testing.assert_array_equal(O.cfg_combine(bank[:B], bank[B:], np.float32(7.5)), g["cfg/noise"])
    both = O.to_noise(ns, "v", np.concatenate([x, x]), bank, t)
    assert rel_err(O.cfg_combine(both[:B], both[B:], np.float32(7.5)), g["cfg/v"]) < 1e-6
    for scale, tag in ((np.float32(1.0), "big"), (np.float32(0.05), "small")):
        assert rel_err(O.data_prediction(ns, x * scale, bank[:B] * scale, t), g[f"x0/{tag}"]) < 1e-6
        assert rel_err(O.data_prediction(ns, x * scale, bank[:B] * scale, t, (0.995, 1.0)), g[f"x0_thr/{tag}"]) < 1e-6
    # quantile: bit-exact, including the fused lerp rounding
    np.testing.assert_array_equal(O.quantile_abs(g["tiny"] * np.float32(3.0), 0.995), g["tiny_q"])
    np.testing.assert_array_equal(O.dynamic_thresholding(g["tiny"] * np.float32(3.0)), g["tiny_thr"])
    from cases import seeded
    np.testing.assert_array_equal(O.quantile_abs(seeded((3, 3 * 64 * 64), 203).numpy(), 0.995), g["big_q"])
    np.testing.assert_array_equal(seeded(16, 1234).numpy(), g["seed_check"])


@pytest.mark.parametrize("name", [c["name"] for c in SAMPLE_CASES])
def test_sample_loops(golden, name):
    """The oracle's own loops (multistep / singlestep) reproduce the reference: outputs within
    1e-4 relative (numpy transcendental ulps propagate through <= 20 steps; the torch-namespace test
    below is bit-exact), identical call trace."""
    g = golden["samples"]
    case = CASES[name]
    y, inter, calls = run_oracle_case(case, golden["schedules"])
    assert [c[1][0] for c in calls] == g[f"{name}/calls_b"].tolist()
    np.testing.assert_allclose(np.asarray([c[0] for c in calls]), g[f"{name}/calls_t"], rtol=2e-4, atol=1e-3)
    assert rel_err(y, g[f"{name}/y"]) < 1e-4


@pytest.mark.parametrize("name", ["pp2m", "pp3m", "eps3s", "eps3s_cfg", "pp2m_logsnr", "pp3s_taylor", "eps2m_taylor", "pp2m_v"])
def test_sample_loops_torch_namespace_bit_exact(golden, name):
    g = golden["samples"]
    y, _, calls = run_oracle_case(CASES[name], xp=TH)
    np.testing.assert_array_equal(y.numpy(), g[f"{name}/y"])
    np.testing.assert_array_equal(np.asarray([c[0] for c in calls], dtype=np.float32), g[f"{name}/calls_t"])


def _quantile_rows(rs):
    """|x0| rows whose order statistics are non-finite, tied or degenerate, each row as long as the others."""
    n = 11
    rows = []
    for k in range(1, n + 1):                                   # k of the n values +inf, the rest 1
        rows.append(np.r_[np.ones(n - k), np.full(k, np.inf)])
    rows.append(np.r_[rs.randn(n - 2), np.inf, -np.inf])        # |.| turns -inf into +inf
    rows.append(np.r_[rs.randn(n - 1), np.nan])
    rows.append(np.r_[np.nan, np.full(n - 1, np.inf)])
    rows.append(np.full(n, np.nan))
    rows.append(np.round(rs.randn(n) * 2) / 4)                  # heavy ties
    rows.append(np.full(n, 0.75))                               # constant
    rows.append(np.zeros(n))
    rows.append(np.r_[np.zeros(n - 1), np.inf])
    rows.append(np.r_[np.full(n - 1, 3.0e38), -3.4028235e38])   # finite extremes: hi - lo stays finite
    rows += [rs.randn(n) * s for s in (1e-30, 1.0, 1e30)]
    return np.asarray(rows, dtype=np.float32)


def test_quantile_abs_matches_torch_on_non_finite_rows():
    """quantile_abs == torch.quantile(|x|, q, dim=1) bit for bit (NaN equal to NaN) where order statistics are
    infinite: for nine 1s and two +inf (n = 11) q = 0.93 lerps between two infs, 0.90 lands on an inf with w = 0,
    0.87 and 0.83 lerp from 1 to inf with w >= 0.5 (inf - inf: NaN) and w < 0.5 (inf). Plus NaN rows, ties,
    constants, zeros and q in {0, 1}. Every q is used with every row, so each +inf count meets each case."""
    rs = np.random.RandomState(17)
    x = _quantile_rows(rs)
    a = np.abs(x)
    for q in (0.93, 0.90, 0.87, 0.83, 0.0, 1.0, 0.995, 0.5, 0.05, 0.31):
        with np.errstate(invalid="ignore"):
            got = O.quantile_abs(x, q)
        want = torch.quantile(torch.from_numpy(a), q, dim=1).numpy()
        np.testing.assert_array_equal(got, want, err_msg=f"q={q}")
        assert got.dtype == np.float32
    # the table's four cases on the row of nine 1s and two infs
    row = np.r_[np.ones(9), np.full(2, np.inf)].astype(np.float32)[None]
    assert [str(O.quantile_abs(row, q)[0]) for q in (0.93, 0.90, 0.87, 0.83)] == ["nan", "nan", "nan", "inf"]
    # the floor keeps NaN (torch.maximum), so dynamic thresholding turns that whole sample into NaN
    with np.errstate(invalid="ignore"):
        thr = O.dynamic_thresholding(np.r_[np.ones(9), np.full(2, np.inf)].astype(np.float32)[None], 0.87, 1.0)
    assert np.isnan(thr).all()


def test_fma32_follows_ieee_on_non_finite_operands():
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    one = np.float32(1)
    cases = [((one, inf, one), inf), ((np.float32(0), inf, one), nan), ((np.float32(-0.13), inf, inf), nan),
             ((np.float32(0.5), one, inf), inf), ((one, one, nan), nan), ((np.float32(-1), inf, -inf), -inf),
             ((np.float32(3e38), np.float32(2), np.float32(0)), inf),            # finite operands, overflowing result
             ((np.float32(3.4028235e38), one, np.float32(2.0 ** 103)), inf),    # exactly halfway to 2^128: to even (inf)
             ((np.float32(3.4028235e38), one, np.float32(2.0 ** 102)), np.float32(3.4028235e38))]
    for (a, b, c), want in cases:
        got = O._fma32(a, b, c)
        assert got.dtype == np.float32
        assert got.tobytes() == np.float32(want).tobytes() or (np.isnan(got) and np.isnan(want)), (a, b, c, got)
