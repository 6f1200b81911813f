"""SDE-DPM-Solver++ (`DPM_Solver(..., algorithm_type="sde-dpmsolver++")`) on the CPU: the product's host logic on the
numpy executor (tests/sde_oracle.py). eta = 0 against the ODE run bit for bit; the product against k-diffusion's
DPM++ 2M / 3M SDE loops in float64 fed the same noise; the marginals of point-mass data after every update; the final
spread of Gaussian data; the generator's state; the plan's cz through the sharded-plan packing; the rejections."""
import math

import numpy as np
import pytest
import torch

from sde_oracle import SdeOracle, kdiff_sde

SHAPE = (4, 3, 8, 8)


@pytest.fixture()
def sde_backend():
    from dpm_solver_b200 import ops
    be = SdeOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def schedule(name):
    from dpm_solver_b200 import NoiseScheduleFlow, NoiseScheduleVP
    if name == "discrete":
        return NoiseScheduleVP("discrete", betas=torch.linspace(1e-4, 2e-2, 1000))
    if name == "linear":
        return NoiseScheduleVP("linear")
    return NoiseScheduleFlow(shift=3.0)


# time-independent networks, linear in x, one per parameterisation; x0_of(out, x, alpha, sigma) is the data
# prediction the parameterisation makes of the output (float64)
NETS = {
    "noise": (lambda x: 0.3 * x + 0.1, lambda o, x, a, s: (x - s * o) / a),
    "x_start": (lambda x: 0.5 * x - 0.2, lambda o, x, a, s: o),
    "v": (lambda x: 0.2 * x + 0.05, lambda o, x, a, s: a * x - s * o),
    "flow": (lambda x: 0.4 * x - 0.3, lambda o, x, a, s: x - s * o),
}
CASES = [("discrete", "noise"), ("linear", "x_start"), ("discrete", "v"), ("flow", "flow")]


def solver(ns, model_type, net=None, algorithm_type="sde-dpmsolver++", **kw):
    from dpm_solver_b200 import DPM_Solver, model_wrapper
    f = NETS[model_type][0] if net is None else net
    fn = model_wrapper(lambda x, t: f(x), ns, model_type=model_type)
    return DPM_Solver(fn, ns, algorithm_type=algorithm_type, **kw)


def x_T(seed=0, shape=SHAPE):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("sched,model_type", CASES)
@pytest.mark.parametrize("order,solver_type", [(1, "dpmsolver"), (2, "dpmsolver"), (2, "taylor"), (3, "dpmsolver"),
                                               (3, "taylor")])
def test_eta_zero_is_the_ode_run(sde_backend, sched, model_type, order, solver_type):
    ns = schedule(sched)
    x = x_T(1)
    ode = solver(ns, model_type, algorithm_type="dpmsolver++").sample(x, steps=6, order=order, solver_type=solver_type)
    g = torch.Generator().manual_seed(5)
    before = g.get_state()
    for kw in ({"eta": 0.0, "generator": g}, {"eta": 0}):
        sde = solver(ns, model_type).sample(x, steps=6, order=order, solver_type=solver_type, **kw)
        assert torch.equal(sde, ode)
    assert torch.equal(g.get_state(), before)
    assert not sde_backend.draws


@pytest.mark.parametrize("sched,model_type", CASES)
@pytest.mark.parametrize("order,solver_type", [(1, "dpmsolver"), (2, "dpmsolver"), (2, "taylor"), (3, "taylor")])
@pytest.mark.parametrize("eta", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("skip_type", ["time_uniform", "logSNR", "karras"])
def test_matches_k_diffusion_float64(sde_backend, sched, model_type, order, solver_type, eta, skip_type):
    from dpm_solver_b200 import plan as P
    ns = schedule(sched)
    steps = 8
    s = solver(ns, model_type)
    g = torch.Generator().manual_seed(11)
    x = x_T(2)
    out, inter = s.sample(x, steps=steps, order=order, solver_type=solver_type, skip_type=skip_type,
                          lower_order_final=False, eta=eta, generator=g, return_intermediate=True)
    assert len(sde_backend.draws) == steps
    t_0, t_T = 1. / ns.total_N, ns.T
    ts = s.get_time_steps(skip_type=skip_type, t_T=t_T, t_0=t_0, N=steps, device="cpu")
    M = P.Marginals(ns, ts)
    al, sg = M.alpha.double().numpy(), M.sigma.double().numpy()
    ale = M.alpha_e.double().numpy()
    f, x0_of = NETS[model_type]

    def denoise(xv, i):
        return x0_of(f(xv), xv, ale[i], sg[i])

    ref = kdiff_sde(x.double().numpy(), denoise, al, sg, [z.double().numpy() for z in sde_backend.draws], eta, order,
                    solver_type)
    for got, want in zip(inter, ref):
        err = np.abs(got.double().numpy() - want).max() / np.abs(want).max()
        assert err < 2e-5, err


@pytest.mark.parametrize("order,solver_type", [(1, "dpmsolver"), (2, "dpmsolver"), (2, "taylor"), (3, "taylor")])
@pytest.mark.parametrize("eta", [0.5, 1.0, 2.0])
def test_point_mass_keeps_the_marginal(sde_backend, order, solver_type, eta):
    """Data at mu: the network returns x0 = mu, the differences of buffered values vanish, and every update keeps
    x_t ~ N(alpha_t*mu, sigma_t^2) exactly, for any order, eta and step size."""
    from dpm_solver_b200 import plan as P
    ns = schedule("discrete")
    mu, n, steps = 0.7, 1 << 20, 6
    s = solver(ns, "x_start", net=lambda x: torch.full_like(x, mu))
    ts = s.get_time_steps(skip_type="time_uniform", t_T=ns.T, t_0=1. / ns.total_N, N=steps, device="cpu")
    M = P.Marginals(ns, ts)
    al, sg = M.alpha.double().tolist(), M.sigma.double().tolist()
    g = torch.Generator().manual_seed(3)
    x = al[0] * mu + sg[0] * torch.randn((1, n), generator=g, dtype=torch.float64)
    _, inter = s.sample(x.float(), steps=steps, order=order, solver_type=solver_type, eta=eta, generator=g,
                        return_intermediate=True)
    for i, v in enumerate(inter):
        v = v.double()
        se = sg[i] / math.sqrt(n)
        assert abs(v.mean().item() - al[i] * mu) < 6 * se
        assert abs(v.std().item() - sg[i]) < 6 * sg[i] / math.sqrt(2 * n)


@pytest.mark.parametrize("order,solver_type", [(2, "dpmsolver"), (2, "taylor"), (3, "taylor")])
def test_gaussian_data_final_spread(sde_backend, order, solver_type):
    """Data N(0, s_d^2) with its analytic denoiser: a 50-step run ends with the data's spread (a sign error in c1 or c2
    moves it by far more)."""
    ns = schedule("linear")
    sd = 0.5

    def net(x, t):
        a = ns.marginal_alpha(t).reshape(-1, 1)
        s = ns.marginal_std(t).reshape(-1, 1)
        return a * sd ** 2 * x / (a * a * sd ** 2 + s * s)

    from dpm_solver_b200 import DPM_Solver, model_wrapper
    fn = model_wrapper(net, ns, model_type="x_start")
    g = torch.Generator().manual_seed(4)
    x = torch.randn((1, 1 << 18), generator=g)
    out = DPM_Solver(fn, ns, algorithm_type="sde-dpmsolver++").sample(x, steps=50, order=order,
                                                                       solver_type=solver_type, eta=1.0, generator=g,
                                                                       skip_type="logSNR")
    assert abs(out.std().item() / sd - 1) < 0.03


def test_generator_state_follows_normal_calls(sde_backend):
    ns = schedule("discrete")
    g = torch.Generator().manual_seed(9)
    x = x_T(3)
    hook_draws = []

    def xt_fn(xt, t, step):
        hook_draws.append(torch.randn(2, generator=g))     # another consumer of the generator, in program order
        return xt

    s = solver(ns, "noise", correcting_xt_fn=xt_fn)
    s.sample(x, steps=5, order=2, eta=1.0, generator=g)
    g2 = torch.Generator().manual_seed(9)
    expect = [torch.randn(2, generator=g2)]                 # (the hook also runs at the initial state)
    for i in range(5):
        torch.empty_like(x, dtype=torch.float32).normal_(generator=g2)
        expect.append(torch.randn(2, generator=g2))
    assert torch.equal(g.get_state(), g2.get_state())
    assert all(torch.equal(a, b) for a, b in zip(hook_draws, expect))


def test_denoise_to_zero_draws_nothing_more(sde_backend):
    ns = schedule("discrete")
    s = solver(ns, "noise")
    s.sample(x_T(4), steps=4, order=2, eta=1.0, denoise_to_zero=True)
    assert len(sde_backend.draws) == 4


def test_thresholding_and_hooks_run(sde_backend):
    ns = schedule("discrete")
    x = x_T(6)
    for kw in ({"correcting_x0_fn": "dynamic_thresholding"}, {"correcting_x0_fn": lambda x0, t: x0 * 0.9}):
        s = solver(ns, "noise", **kw)
        out = s.sample(x, steps=5, order=3, eta=1.0, generator=torch.Generator().manual_seed(1))
        assert torch.isfinite(out).all()


def test_plan_cache_keys_eta(sde_backend):
    ns = schedule("discrete")
    s = solver(ns, "noise")
    x = x_T(7)
    a = s.sample(x, steps=4, eta=0.5, generator=torch.Generator().manual_seed(2))
    b = s.sample(x, steps=4, eta=1.5, generator=torch.Generator().manual_seed(2))
    c = solver(ns, "noise").sample(x, steps=4, eta=1.5, generator=torch.Generator().manual_seed(2))
    assert not torch.equal(a, b) and torch.equal(b, c)


def test_sharded_plan_carries_cz():
    from dpm_solver_b200 import plan as P
    from dpm_solver_b200.distributed import pack_plan, unpack_plan
    ns = schedule("discrete")
    ts = torch.linspace(1., 1e-3, 9)
    plan = P.multistep_plan(ns, "dpmsolver++", "taylor", ts, 3, False, eta=1.0)
    assert all(c.cz > 0 for c in plan)
    assert [c.__dict__ for c in unpack_plan(pack_plan(plan))] == [c.__dict__ for c in plan]


def test_rejections(sde_backend):
    from dpm_solver_b200 import DPM_Solver, UniPC, model_wrapper
    ns = schedule("discrete")
    calls = []

    def net(x, t, *a):
        calls.append(1)
        return x

    x = x_T(8)
    s = solver(ns, "noise", net=net)
    for kw in ({"method": "singlestep"}, {"method": "singlestep_fixed"}, {"method": "adaptive"}, {"eta": -1.0},
               {"eta": float("nan")}, {"eta": float("inf")}, {"eta": "1"}, {"generator": "cpu"}):
        with pytest.raises(ValueError):
            s.sample(x, steps=4, **kw)
    with pytest.raises(ValueError):
        s.inverse(x, steps=4)
    t = torch.tensor([0.5])
    for call in (lambda: s.dpm_solver_first_update(x, t, t * 0.5),
                 lambda: s.multistep_dpm_solver_second_update(x, [x, x], [t, t * 0.8], t * 0.5),
                 lambda: s.multistep_dpm_solver_third_update(x, [x, x, x], [t, t * 0.9, t * 0.8], t * 0.5),
                 lambda: s.multistep_dpm_solver_update(x, [x, x], [t, t * 0.8], t * 0.5, 2),
                 lambda: s.singlestep_dpm_solver_update(x, t, t * 0.5, 2),
                 lambda: s.singlestep_dpm_solver_second_update(x, t, t * 0.5),
                 lambda: s.singlestep_dpm_solver_third_update(x, t, t * 0.5)):
        with pytest.raises(ValueError):
            call()
    ode = solver(ns, "noise", net=net, algorithm_type="dpmsolver++")
    for kw in ({"eta": 1.0}, {"generator": torch.Generator()}):
        with pytest.raises(ValueError):
            ode.sample(x, steps=4, **kw)
    fn = model_wrapper(net, ns)
    with pytest.raises(ValueError):
        UniPC(fn, ns, algorithm_type="sde-dpmsolver++")
    with pytest.raises(ValueError):
        DPM_Solver(fn, ns, algorithm_type="sde-dpmsolver++", reference_rounding=True)
    uc, c1, c2 = torch.zeros(4), torch.ones(4), 2 * torch.ones(4)
    for kw in ({"condition": [c1, c2], "guidance_scale": [2.0, 1.5]},
               {"condition": [c1, c2], "guidance_scale": [2.0, 1.5], "perp_neg": True},
               {"condition": c1, "guidance_scale": 2.0, "apg_eta": 0.0},
               {"condition": c1, "guidance_scale": 2.0, "cfg_pp": True},
               {"condition": [c1], "guidance_scale": [2.0], "guidance_mask": [torch.ones(8, 8)]}):
        with pytest.raises(ValueError):
            w = model_wrapper(net, ns, guidance_type="classifier-free", unconditional_condition=uc, **kw)
            DPM_Solver(w, ns, algorithm_type="sde-dpmsolver++")
    assert not calls and not sde_backend.draws
