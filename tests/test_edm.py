"""EDM-preconditioned sampling (`NoiseScheduleEDM`, `model_wrapper(..., model_type="edm")`) and skip_type="karras" on
the CPU: the schedule's scalars and conversion words against 50-digit mpmath, the Karras grids against their fp64
definitions, and the product's host logic on the numpy executor against the UNMODIFIED reference solver driven on the
EDM schedule (tests/edm_oracle.py), bit for bit; UniPC against the fp64 transcription of unipc_oracle; second-order
convergence on a Gaussian problem with a closed-form solution."""
import itertools
import math
import random
from unittest import mock

import numpy as np
import pytest
import torch

from cases import exact_net, make_betas, seeded
from oracle import ref_loader

mpmath = pytest.importorskip("mpmath")
needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
B, SHAPE = 3, (3, 2, 4, 4)
SCHEDULES = [dict(), dict(sigma_min=0.002, sigma_max=80., sigma_data=1.0), dict(sigma_min=0.03, sigma_max=14.6,
                                                                              sigma_data=0.5, rho=5., total_N=50)]


def schedule(**kw):
    from dpm_solver_b200 import NoiseScheduleEDM
    return NoiseScheduleEDM(**kw)


def ulps(a, b64):
    """|a - b| in units of the fp32 spacing at b."""
    b32 = np.asarray(b64).astype(np.float32)
    sp = np.spacing(np.abs(b32)).astype(np.float64)
    return np.abs(np.asarray(a, dtype=np.float64) - b64) / np.maximum(sp, 1e-300)


def mp_eval(fn, xs):
    mpmath.mp.dps = 50
    return np.array([float(fn(mpmath.mpf(float(v)))) for v in xs])


# ---- 1. the schedule ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw", SCHEDULES)
def test_schedule_scalars_match_mpmath(kw):
    ns = schedule(**kw)
    mp = mpmath
    mp.mp.dps = 50
    smin, smax, sd = mp.mpf(ns.sigma_min), mp.mpf(ns.sigma_max), mp.mpf(ns.sigma_data)
    rho, N = mp.mpf(ns.rho), ns.total_N
    c = mp.mpf(float(np.float32(1. / N)))
    t = torch.linspace(float(np.float32(1. / N)), 1., 2001)

    def sig(tt):
        u = (tt - c) / (1 - c)
        return (smin ** (1 / rho) + u * (smax ** (1 / rho) - smin ** (1 / rho))) ** rho
    s32 = ns.sigma(t)
    # end to end: u, the ramp and the power each round; the power multiplies the ramp's relative error by rho (measured:
    # at most 13.8 ulp at rho = 7)
    assert ulps(s32.numpy(), mp_eval(sig, t)).max() <= 3 * ns.rho
    # each later quantity against the exact function of the fp32 noise level it is computed from
    s = s32.double().numpy()
    r = lambda v: mp.sqrt(v * v + sd * sd)
    al, sg, la, lm = (f(t) for f in (ns.marginal_alpha, ns.marginal_std, ns.marginal_log_mean_coeff, ns.marginal_lambda))
    # (three and four rounded ops; measured at most 1.97 and 1.73 ulp)
    assert ulps(al.numpy(), mp_eval(lambda v: 1 / r(v), s)).max() <= 2.5
    assert ulps(sg.numpy(), mp_eval(lambda v: v / r(v), s)).max() <= 2.5
    assert np.abs(la.double().numpy() - mp_eval(lambda v: -mp.log(r(v)), s)).max() <= 2 * np.spacing(np.float32(8.))
    assert ulps(lm.numpy(), mp_eval(lambda v: -mp.log(v), s)).max() <= 1
    assert torch.equal(ns.model_input_time(t), 0.25 * torch.log(s32))
    got = ns.marginals(t)
    for g, w in zip(got, (la, sg, lm, al)):
        assert torch.equal(g, w)
    # the conversion words at the fp32 marginals: each formed in double and rounded once
    for x0 in (True, False):
        w = [ns.conversion_words(float(a), float(g), x0) for a, g in zip(al[::40], sg[::40])]
        a64, g64 = al[::40].double().numpy(), sg[::40].double().numpy()
        if x0:
            want = [(sd * sd * mp.mpf(a), sd * mp.mpf(g)) for a, g in zip(a64, g64)]
        else:
            want = [(mp.mpf(g), -sd * mp.mpf(a)) for a, g in zip(a64, g64)]
        for k in range(2):
            got_k = np.array([v[k] for v in w])
            assert np.array_equal(got_k, got_k.astype(np.float32).astype(np.float64))
            assert ulps(got_k, np.array([float(v[k]) for v in want])).max() <= 0.5 + 1e-6


@pytest.mark.parametrize("kw", SCHEDULES)
def test_inverse_lambda_round_trip(kw):
    ns = schedule(**kw)
    t = torch.linspace(float(np.float32(1. / ns.total_N)), 1., 2001)
    back = ns.inverse_lambda(ns.marginal_lambda(t))
    # dt/dlambda = -s*dt/ds: an ulp of lambda and the fp32 powers move t by a few 1e-7
    assert (back - t).abs().max() <= 2e-6


def test_time_uniform_steps_are_the_karras_grid():
    from dpm_solver_b200 import DPM_Solver
    for kw, n in itertools.product(SCHEDULES, (5, 18, 50)):
        ns = schedule(**kw)
        s = DPM_Solver(lambda x, t: x, ns)
        ts = s.get_time_steps("time_uniform", ns.T, 1. / ns.total_N, n, "cpu")
        i = np.arange(n + 1) / n
        a, b = ns.sigma_max ** (1 / ns.rho), ns.sigma_min ** (1 / ns.rho)
        want = (a + i * (b - a)) ** ns.rho
        got = ns.sigma(ts).double().numpy()
        assert np.abs(got / want - 1).max() <= 8 * ns.rho * 2 ** -24, (kw, n)
        assert float(ns.sigma(torch.tensor([1.]))) == pytest.approx(ns.sigma_max, rel=4 * ns.rho * 2 ** -24)
        assert float(ns.sigma(ts[-1:])) == pytest.approx(ns.sigma_min, rel=4 * ns.rho * 2 ** -24)


def _karras_schedules():
    from dpm_solver_b200 import NoiseScheduleFlow, NoiseScheduleVP
    return {"discrete": NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1])),
            "linear": NoiseScheduleVP("linear"), "cosine": NoiseScheduleVP("cosine"),
            "flow": NoiseScheduleFlow(shift=3.0), "edm": schedule()}


@pytest.mark.parametrize("name", ["discrete", "linear", "cosine", "flow", "edm"])
def test_karras_grid_matches_its_fp64_definition(name):
    from dpm_solver_b200 import DPM_Solver, UniPC
    ns = _karras_schedules()[name]
    t_T, t_0 = ns.T, 1. / ns.total_N
    for n in (1, 7, 20, 50):
        ts = DPM_Solver(lambda x, t: x, ns).get_time_steps("karras", t_T, t_0, n, "cpu")
        assert torch.equal(ts, UniPC(lambda x, t: x, ns).get_time_steps("karras", t_T, t_0, n, "cpu"))
        assert ts.dtype == torch.float32 and ts.shape == (n + 1,)
        lT = float(ns.marginal_lambda(torch.tensor(t_T)))
        l0 = float(ns.marginal_lambda(torch.tensor(t_0)))
        r64 = np.linspace(math.exp(-lT / 7), math.exp(-l0 / 7), n + 1) ** 7
        lam64 = -np.log(r64)
        lam = ns.marginal_lambda(ts).double().numpy()
        # lambda of the returned labels: the fp32 ramp, power, log, inverse_lambda and marginal_lambda each round;
        # on the tabulated VP schedule the piecewise-linear inverse and forward maps agree to a few 1e-6
        assert np.abs(lam - lam64).max() <= 2e-4 * max(1., np.abs(lam64).max()), (name, n)
        assert np.all(np.diff(ts.numpy()) < 0), (name, n)


def test_singlestep_orders_take_the_karras_grid():
    from dpm_solver_b200 import DPM_Solver
    ns = schedule()
    s = DPM_Solver(lambda x, t: x, ns)
    outer, orders = s.get_orders_and_timesteps_for_singlestep_solver(10, 3, "karras", ns.T, 1. / ns.total_N, "cpu")
    full = s.get_time_steps("karras", ns.T, 1. / ns.total_N, 10, "cpu")
    assert torch.equal(outer, full[torch.cumsum(torch.tensor([0] + orders), 0)])


def test_defaults_and_validation():
    ns = schedule()
    assert ns.schedule == "edm" and ns.T == 1. and ns.total_N == 1000
    assert (ns.sigma_min, ns.sigma_max, ns.sigma_data, ns.rho) == (0.002, 80., 0.5, 7.)
    for bad in (dict(sigma_min=0.), dict(sigma_min=-1.), dict(sigma_min=90.), dict(sigma_max=float("inf")),
                dict(sigma_max=float("nan")), dict(sigma_data=0.), dict(sigma_data=float("inf")), dict(rho=0.),
                dict(rho=-7.), dict(rho=float("nan")), dict(total_N=1), dict(total_N=2.5)):
        with pytest.raises(ValueError):
            schedule(**bad)


# ---- 2. rejections -----------------------------------------------------------------------------------------------------

def test_rejections_raise_before_any_launch():
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops

    class NoLaunch:
        def __getattr__(self, name):
            raise AssertionError("the executor was reached: " + name)

    old = ops._backend
    ops.set_backend(NoLaunch())
    try:
        edm, vp, flow = schedule(), new.NoiseScheduleVP("linear"), new.NoiseScheduleFlow(shift=3.0)
        net = lambda x, t: x
        for other in (vp, flow):
            with pytest.raises(ValueError, match="NoiseScheduleEDM"):
                new.model_wrapper(net, other, model_type="edm")
        for mt in ("noise", "x_start", "v", "score", "flow"):
            with pytest.raises(ValueError, match="model_type='edm' only|needs a NoiseScheduleFlow"):
                new.model_wrapper(net, edm, model_type=mt)
        with pytest.raises(ValueError, match="classifier guidance"):
            new.model_wrapper(net, edm, model_type="edm", guidance_type="classifier", classifier_fn=net)
        fn = new.model_wrapper(net, edm, model_type="edm")
        with pytest.raises(ValueError, match="reference_rounding"):
            new.DPM_Solver(fn, edm, reference_rounding=True)
        with pytest.raises(ValueError, match="Unsupported skip_type"):
            new.DPM_Solver(fn, edm).get_time_steps("karass", 1., 1e-3, 4, "cpu")
        new.DPM_Solver(fn, edm)
        new.UniPC(fn, edm)
    finally:
        ops.set_backend(old)


# ---- 3. the unmodified reference solver as the oracle -----------------------------------------------------------------

def edm_net(calls=None):
    """Exact IEEE multiplies and adds; the conditional blocks differ in scale and offset."""
    def net(x, t, c=None):
        if calls is not None:
            calls.append((tuple(x.shape), t.tolist()))
        out = exact_net(x.float(), t)
        if c is not None:
            out = out * (1. + 0.3 * c.reshape(-1, 1, 1, 1)) + 0.05 * c.reshape(-1, 1, 1, 1)
        return out
    return net


GUIDANCE = {
    "none": None,
    "scalar": dict(kind="scalar", scales=3.5, K=1),
    "per_sample": dict(kind="per_sample", scales=[7.5, 1.0, -2.0], K=1),
    "multi2": dict(kind="multi", scales=[7.5, -2.0], K=2),
    "multi3": dict(kind="multi", scales=[4.0, 0.0, -1.5], K=3),
}


def make_pair(algo, thr, guidance, phi=0.0, sched=None):
    """(reference solver, product solver, reference calls, product calls)."""
    import dpm_solver_b200 as new
    import edm_oracle as E
    kw = sched or {}
    rns, pns = E.reference_schedule(**kw), schedule(**kw)
    rc, pc = [], []
    g = GUIDANCE[guidance]
    uc = torch.zeros(B, 1)
    if g is None:
        rs = E.reference_solver(edm_net(), rns, algo, thr, calls=rc)
        pfn = new.model_wrapper(edm_net(pc), pns, model_type="edm")
    else:
        conds = [torch.full((B, 1), float(k + 1)) for k in range(g["K"])]
        rs = E.reference_solver(edm_net(), rns, algo, thr, calls=rc, phi=phi,
                                guidance=dict(uc=uc, conds=conds, scales=g["scales"], kind=g["kind"]))
        pfn = new.model_wrapper(edm_net(pc), pns, model_type="edm", guidance_type="classifier-free",
                                condition=conds if g["kind"] == "multi" else conds[0], unconditional_condition=uc,
                                guidance_scale=g["scales"], guidance_rescale=phi)
    ps = new.DPM_Solver(pfn, pns, algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
    return rs, ps, rc, pc


@pytest.fixture()
def edm_backend():
    from dpm_solver_b200 import ops
    import edm_oracle as E
    be = E.EDMOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2), ("singlestep", 3),
           ("singlestep_fixed", 2), ("singlestep_fixed", 3)]
SKIPS = ["time_uniform", "logSNR", "time_quadratic", "karras"]


def sweep():
    """A seeded sweep of algorithm x method x order x skip type x schedule x guidance x thresholding: the full product
    of algorithm, method and guidance, the rest drawn."""
    rng = random.Random(20260)
    out = []
    for algo, (method, order), guidance in itertools.product(("dpmsolver++", "dpmsolver"), METHODS, GUIDANCE):
        thr = algo == "dpmsolver++" and rng.random() < 0.5
        out.append((algo, method, order, rng.choice(SKIPS), rng.randrange(len(SCHEDULES)), guidance, thr,
                    rng.choice(["dpmsolver", "taylor"]), rng.random() < 0.3))
    return out


@needs_ref
@pytest.mark.parametrize("algo,method,order,skip,sched,guidance,thr,solver_type,d2z", sweep())
def test_sample_matches_reference_solver(edm_backend, algo, method, order, skip, sched, guidance, thr, solver_type, d2z):
    rs, ps, rc, pc = make_pair(algo, thr, guidance, sched=SCHEDULES[sched])
    x = seeded(SHAPE, 11) * float(ps.noise_schedule.marginal_std(torch.tensor([1.])))
    kw = dict(steps=7, order=order, method=method, skip_type=skip, solver_type=solver_type, denoise_to_zero=d2z,
              return_intermediate=True)
    yr, ir = rs.sample(x.clone(), **kw)
    yp, ip = ps.sample(x.clone(), **kw)
    assert pc == rc                                  # the same (x.shape, c_noise) network calls, in the same order
    assert len(ip) == len(ir)
    for a, b in zip(ip, ir):
        np.testing.assert_array_equal(a.numpy(), b.numpy())
    np.testing.assert_array_equal(yp.numpy(), yr.numpy())
    assert yp.isfinite().all()


@needs_ref
@pytest.mark.parametrize("algo,thr", [("dpmsolver++", False), ("dpmsolver++", True), ("dpmsolver", False)])
@pytest.mark.parametrize("method,order", [("multistep", 2), ("singlestep", 3)])
def test_guidance_rescale_matches_reference_solver(edm_backend, algo, thr, method, order):
    """combine and rescale the raw network outputs, then convert (the ratio in fp64 on both sides)."""
    rs, ps, rc, pc = make_pair(algo, thr, "scalar", phi=0.7)
    x = seeded(SHAPE, 5) * 80.
    kw = dict(steps=6, order=order, method=method)
    yr, yp = rs.sample(x.clone(), **kw), ps.sample(x.clone(), **kw)
    assert pc == rc and ("ratio", 2) in edm_backend.log
    np.testing.assert_array_equal(yp.numpy(), yr.numpy())


@needs_ref
@pytest.mark.parametrize("algo", ["dpmsolver++", "dpmsolver"])
@pytest.mark.parametrize("order", [2, 3])
def test_adaptive_matches_reference_solver(edm_backend, algo, order):
    """The host controller (EDM has no device controller kind)."""
    from dpm_solver_b200 import ops
    assert "edm" not in ops.AdaptiveController.SUPPORTED
    rs, ps, rc, pc = make_pair(algo, False, "scalar")
    x = seeded(SHAPE, 7)
    kw = dict(order=order, method="adaptive", atol=0.05, rtol=0.1)
    nfe = []
    for s in (rs, ps):
        with mock.patch("builtins.print") as pr:
            y = s.sample(x.clone(), **kw)
            nfe.append((pr.call_args[0][-1], y))
    assert nfe[0][0] == nfe[1][0] and len(pc) == len(rc)
    yr, yp = nfe[0][1].numpy(), nfe[1][1].numpy()
    # the error estimate is a mean whose summation order differs from torch's (DESIGN.md section 2)
    assert np.abs(yp.astype(np.float64) - yr).max() / np.abs(yr).max() <= 1e-5


@needs_ref
def test_model_fn_direct_call_returns_eps(edm_backend):
    """WrappedModel.__call__ returns eps = sigma_t*y - (sd*alpha_t)*F, with one time label for the batch and one per
    sample."""
    rs, ps, _, _ = make_pair("dpmsolver", False, "scalar")
    x = seeded(SHAPE, 3)
    for t in (torch.full((B,), 0.6), torch.tensor([0.9, 0.5, 0.2])):
        np.testing.assert_array_equal(ps._wrapped(x, t).numpy(), rs.model(x, t).numpy())


def test_network_receives_y_and_c_noise(edm_backend):
    """The first call sees x_T itself (the solver's state is the network input) and every call c_noise = ln(s)/4 of its
    label, one row per input row."""
    import dpm_solver_b200 as new
    ns = schedule()
    seen = []

    def net(x, t, c=None):
        seen.append((x.clone(), t.clone()))
        return exact_net(x, t)
    uc, c = torch.zeros(B, 1), torch.ones(B, 1)
    fn = new.model_wrapper(net, ns, model_type="edm", guidance_type="classifier-free", condition=c,
                           unconditional_condition=uc, guidance_scale=2.0)
    s = new.DPM_Solver(fn, ns)
    x = seeded(SHAPE, 4) * 80.
    steps = 6
    s.sample(x.clone(), steps=steps, order=2, denoise_to_zero=True)
    ts = s.get_time_steps("time_uniform", ns.T, 1. / ns.total_N, steps, "cpu")
    labels = list(ts[:steps]) + [ts[-1]]
    assert len(seen) == steps + 1
    assert torch.equal(seen[0][0][:B], x) and torch.equal(seen[0][0][B:], x)
    for (xin, tin), lab in zip(seen, labels):
        want = 0.25 * torch.log(ns.sigma(lab.reshape(1)))
        assert tin.shape == (2 * B,) and torch.equal(tin, want.expand(2 * B))


@needs_ref
def test_add_noise_inverse_and_diffedit(edm_backend):
    from dpm_solver_b200 import DiffEditCorrector
    rs, ps, _, _ = make_pair("dpmsolver++", False, "none")
    x, noise = seeded(SHAPE, 1), seeded((2,) + SHAPE, 2)
    t = torch.tensor([0.3, 0.8])
    np.testing.assert_array_equal(ps.add_noise(x, t, noise=noise).numpy(), rs.add_noise(x, t, noise=noise).numpy())
    kw = dict(steps=5, order=2)
    np.testing.assert_array_equal(ps.inverse(x.clone(), **kw).numpy(), rs.inverse(x.clone(), **kw).numpy())
    # the corrector re-noises the source to the label's (alpha_t, sigma_t): y = alpha_t*x0 + sigma_t*n
    ns = ps.noise_schedule
    seen = []
    real = edm_backend.diffedit_corrector

    def spy(xx, x0, mask, alpha, sigma, generator=None):
        seen.append((alpha, sigma))
        return real(xx, x0, mask, alpha, sigma, generator=generator)
    edm_backend.diffedit_corrector = spy
    corr = DiffEditCorrector(ns, x, torch.ones(SHAPE[0], 1, 1, 1).round(), generator=torch.Generator().manual_seed(0))
    tl = torch.tensor([0.55])
    corr(x, tl, 0)
    assert seen == [(float(ns.marginal_alpha(tl)), float(ns.marginal_std(tl)))]


# ---- 4. UniPC -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(12))
def test_unipc_follows_the_fp64_transcription(edm_backend, seed):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import plan as P
    from unipc_oracle import unipc_fp64
    rng = random.Random(seed)
    kw = SCHEDULES[rng.randrange(len(SCHEDULES))]
    alg, variant = rng.choice(["dpmsolver++", "dpmsolver"]), rng.choice(["bh1", "bh2"])
    steps = rng.randint(2, 10)
    order, corr, lof = rng.randint(1, min(3, steps)), rng.random() < 0.8, rng.random() < 0.5
    skip = rng.choice(SKIPS)
    ns = schedule(**kw)
    net = lambda x, t: 0.1 * x + ((t * 0.25) - 0.02).reshape(-1, *([1] * (x.dim() - 1)))
    s = new.UniPC(new.model_wrapper(net, ns, model_type="edm"), ns, algorithm_type=alg, variant=variant)
    x = torch.randn(2, 3, 4, generator=torch.Generator().manual_seed(seed)) * float(ns.marginal_std(torch.tensor([1.])))
    y, inter = s.sample(x.clone(), steps=steps, order=order, skip_type=skip, lower_order_final=lof, use_corrector=corr,
                        return_intermediate=True)
    ts = s.get_time_steps(skip, ns.T, 1. / ns.total_N, steps, "cpu")
    marg = P.Marginals(ns, ts)
    lam, al, sg = (v.double().numpy() for v in (marg.lam, marg.alpha, marg.sigma))
    a_e = marg.alpha_e.double().numpy()
    tin = ns.model_input_time(ts).double().numpy()
    sd = ns.sigma_data
    data = alg == "dpmsolver++"

    def model(xx, i):
        F = 0.1 * xx + (tin[i] * 0.25 - 0.02)
        return sd * sd * a_e[i] * xx + sd * sg[i] * F if data else sg[i] * xx - sd * a_e[i] * F

    xN, xs = unipc_fp64(model, al, sg, lam, x.double().numpy(), order, data, variant == "bh2", corr, lof,
                        return_intermediate=True)
    scale = max(1.0, float(np.abs(xN).max()))
    # the plan rounds each step's h = lambda_i - lambda_{i-1} to fp32 (as the reference does); the noise-prediction
    # update multiplies that rounding by e^h, which a few large steps over EDM's lambda range make large
    if not data:
        scale *= math.exp(float(np.abs(np.diff(lam)).max()))
    for k in range(steps + 1):
        assert float(np.abs(inter[k].double().numpy() - xs[k]).max()) <= 1e-5 * scale, (kw, alg, variant, skip, k)


# ---- 5. convergence ----------------------------------------------------------------------------------------------------

def test_dpm_solver_pp_2m_converges_at_order_two(edm_backend):
    """Data x0 ~ N(0, S^2): D(x; s) = S^2/(S^2 + s^2)*x exactly, and the probability-flow ODE carries x_T at s_max to
    x(s) = x_T*sqrt(S^2 + s^2)/sqrt(S^2 + s_max^2). The network returns F = (D - c_skip*x)/c_out at the x = y/c_in it
    is handed; the error of DPM-Solver++ 2M at sigma_min falls by about 4 per doubling of the steps."""
    import dpm_solver_b200 as new
    ns = schedule()
    S, sd = 0.8, ns.sigma_data

    def net(y, c_noise):
        s = torch.exp(4. * c_noise.double()).reshape(-1, *([1] * (y.dim() - 1)))
        r = torch.sqrt(s * s + sd * sd)
        x = y.double() * r
        D = S * S / (S * S + s * s) * x
        return ((D - sd * sd / (r * r) * x) / (s * sd / r)).float()

    s = new.DPM_Solver(new.model_wrapper(net, ns, model_type="edm"), ns, algorithm_type="dpmsolver++")
    yT = torch.linspace(-2., 2., 64).reshape(2, 32)
    smax, smin = float(ns.sigma(torch.tensor([1.]))), float(ns.sigma(torch.tensor([float(np.float32(1e-3))])))
    r = lambda v: math.sqrt(v * v + sd * sd)
    xT = yT.double() * r(smax)
    exact = xT * math.sqrt(S * S + smin * smin) / math.sqrt(S * S + smax * smax) / r(smin)
    errs = []
    for n in (12, 24, 48):
        y = s.sample(yT.clone(), steps=n, order=2, method="multistep", skip_type="time_uniform")
        errs.append(float((y.double() - exact).abs().max()))
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    assert all(3.0 <= q <= 6.0 for q in ratios), (errs, ratios)
