"""UniPC multistep sampling (dpm_solver_b200/unipc.py) on the CPU: the folded words against mpmath, convergence orders
on a problem with a closed-form solution, the reduction to the unmodified reference's DPM-Solver(++)(2M), the product on
the numpy executor against an fp64 transcription of the method, hooks and rejected arguments."""
import math
import random

import numpy as np
import pytest
import torch

from cases import make_betas
from dpm_solver_b200 import NoiseScheduleFlow, NoiseScheduleVP, UniPC, model_wrapper, ops, plan as P
from oracle import ref_loader
from unipc_oracle import (LinearVP64, UniPCOracle, anchor_error, exact_solution, gaussian_x0, ulp32, unipc_fp64,
                          words_mp)

mpmath = pytest.importorskip("mpmath")


@pytest.fixture()
def uni_backend():
    be = UniPCOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def schedule(name):
    if name == "discrete":
        return NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    if name == "flow":
        return NoiseScheduleFlow(shift=3.0)
    return NoiseScheduleVP(name)


# ---- 1. folded words ---------------------------------------------------------------------------------------------------

def _check_words(ns, skip, steps, order, variant, alg, use_corrector, lof):
    s = UniPC(lambda x, t: x, ns, algorithm_type=alg, variant=variant)
    ts = s.get_time_steps(skip, ns.T, 1. / ns.total_N, steps, "cpu")
    marg = P.Marginals(ns, ts)
    ords = P.unipc_orders(steps, order, lof)
    _, launches = P.unipc_plan(alg, variant, marg, ords, use_corrector)
    exact = words_mp(alg, variant, marg.lam.tolist(), marg.alpha.tolist(), marg.sigma.tolist(), ords, use_corrector)
    assert len(launches) == len(exact) == steps - 1
    for i, (w, e) in enumerate(zip(launches, exact)):
        assert (w.pc, w.pp) == ((ords[i] if use_corrector else 0), ords[i + 1])
        got = dict(ct=w.ct, a=w.a, c0=w.c0, cd0=w.cd[0], cd1=w.cd[1], cp0=w.cp[0], cp1=w.cp[1])
        for k, v in got.items():
            ex = e.get(k, 0)
            assert abs(v - float(ex)) <= ulp32(ex), (i, k, v, float(ex))


@pytest.mark.parametrize("sched", ["discrete", "linear", "cosine", "flow"])
@pytest.mark.parametrize("skip", ["logSNR", "time_uniform", "time_quadratic"])
def test_plan_words_within_one_ulp(sched, skip):
    ns = schedule(sched)
    rng = random.Random(hash((sched, skip)) & 0xffff)
    for steps in range(1, 51):
        order = rng.choice([o for o in (1, 2, 3) if o <= steps])
        _check_words(ns, skip, steps, order, rng.choice(["bh1", "bh2"]), rng.choice(["dpmsolver++", "dpmsolver"]),
                     rng.random() < 0.8, rng.random() < 0.5)


@pytest.mark.parametrize("sched", ["discrete", "linear", "cosine", "flow"])
def test_plan_words_within_one_ulp_at_1000_steps(sched):
    """|h| is small: the h_phi recursion cancels in fp64 there, the series does not."""
    for alg, variant in (("dpmsolver++", "bh2"), ("dpmsolver", "bh1")):
        _check_words(schedule(sched), "logSNR" if sched != "cosine" else "time_uniform", 1000, 3, variant, alg, True,
                     True)


def test_orders_lower_the_final_steps_for_every_step_count():
    assert P.unipc_orders(20, 3, True) == [1, 2] + [3] * 16 + [2, 1]
    assert P.unipc_orders(20, 3, False) == [1, 2] + [3] * 18
    assert P.unipc_orders(3, 3, True) == [1, 2, 1]


# ---- 2. convergence anchors ----------------------------------------------------------------------------------------------

ANCHORS = [  # (algorithm, variant, order, corrector) -> |x_N - exact| at N = 10, 20, 40, 80
    (("dpmsolver++", "bh2", 2, True), [1.74e-2, 3.18e-3, 4.35e-4, 5.55e-5]),
    (("dpmsolver++", "bh2", 2, False), [1.11e-2, 4.99e-3, 1.36e-3, 3.45e-4]),
    (("dpmsolver++", "bh2", 1, True), [5.36e-2, 1.58e-2, 4.14e-3, 1.04e-3]),
    (("dpmsolver++", "bh2", 1, False), [8.29e-2, None, None, 1.15e-2]),
    (("dpmsolver++", "bh1", 2, True), [7.23e-2, 7.54e-3, 8.69e-4, 1.03e-4]),
    (("dpmsolver", "bh2", 2, True), [2.23e-2, 3.31e-3, 4.41e-4, 5.60e-5]),
    (("dpmsolver", "bh1", 3, True), [1.33e-2, 1.17e-3, 7.27e-5, 4.14e-6]),
]
NS = (10, 20, 40, 80)


def _close(got, want, digits):
    return abs(got - want) <= 0.5 * 10 ** (math.floor(math.log10(want)) - digits + 1) + 1e-15


@pytest.mark.parametrize("cfg,errs", ANCHORS)
def test_fp64_transcription_reproduces_the_anchors(cfg, errs):
    alg, variant, order, corr = cfg
    got = [anchor_error(N, order, alg == "dpmsolver++", variant == "bh2", corr) for N in NS]
    for g, w in zip(got, errs):
        if w is not None:
            assert _close(g, w, 3), (got, errs)
    slope = math.log2(got[2] / got[3])
    assert slope >= order + 0.8 if corr else abs(slope - order) < 0.2, slope


def product_error(N, alg, variant, order, corr):
    """|x_N - exact| of the product on the numpy executor, fp32, linear VP, logSNR grid."""
    ns = NoiseScheduleVP("linear")

    def net(x, t):          # the exact x0 of the Gaussian problem, as an x_start network
        al, sg = ns.marginal_alpha(t).reshape(-1, 1), ns.marginal_std(t).reshape(-1, 1)
        return 0.5 + al * 0.09 / (al * al * 0.09 + sg * sg) * (x - al * 0.5)

    fn = model_wrapper(net, ns, model_type="x_start")
    x = torch.full((1, 8), 1.3)
    y = UniPC(fn, ns, algorithm_type=alg, variant=variant).sample(x, steps=N, t_start=1., t_end=1e-3, order=order,
                                                                   skip_type="logSNR", lower_order_final=False,
                                                                   use_corrector=corr)
    vp = LinearVP64()
    ex = exact_solution(1.3, vp.alpha(1.), vp.sigma(1.), vp.alpha(1e-3), vp.sigma(1e-3))
    return abs(float(y[0, 0]) - ex)


@pytest.mark.parametrize("cfg,errs", ANCHORS)
def test_product_on_the_executor_reproduces_the_anchors(uni_backend, cfg, errs):
    alg, variant, order, corr = cfg
    got = [product_error(N, alg, variant, order, corr) for N in NS]
    for g, w in zip(got, errs):
        # (2 digits, or 1e-6 where that is finer: fp32 state and marginals of magnitude ~1 over 80 steps do not resolve
        # more, e.g. 4.6e-6 for the order-3 anchor 4.14e-6)
        if w is not None:
            assert _close(g, w, 2) or abs(g - w) <= 1e-6, (got, errs)


# ---- 3. against the unmodified reference ---------------------------------------------------------------------------------

@pytest.mark.skipif(not ref_loader.available(), reason="reference bytecode not built")
@pytest.mark.parametrize("alg", ["dpmsolver++", "dpmsolver"])
@pytest.mark.parametrize("steps", [10, 20])
def test_unip2_bh2_without_corrector_is_the_reference_multistep_2(uni_backend, alg, steps):
    ref = ref_loader.load("dpm_solver_pytorch")
    betas = torch.from_numpy(make_betas("sd")[1])
    net = lambda x, t: 0.1 * x + torch.sin(t * 0.003).reshape(-1, 1, 1, 1) * 0.2 - 0.05 * torch.tanh(x)
    x = torch.randn(2, 3, 8, 8, generator=torch.Generator().manual_seed(5))
    ns_r = ref.NoiseScheduleVP("discrete", betas=betas)
    y_r = ref.DPM_Solver(ref.model_wrapper(net, ns_r), ns_r, algorithm_type=alg).sample(
        x, steps=steps, order=2, method="multistep", lower_order_final=False, skip_type="time_uniform")
    ns = NoiseScheduleVP("discrete", betas=betas)
    y = UniPC(model_wrapper(net, ns), ns, algorithm_type=alg, variant="bh2").sample(
        x, steps=steps, order=2, lower_order_final=False, use_corrector=False)
    rel = float((y - y_r).abs().max() / y_r.abs().max())
    assert rel < 1e-6, rel


# ---- 4. the product against the fp64 transcription ----------------------------------------------------------------------

PARAMS = ["noise", "x_start", "v", "score"]


def draw(rng):
    sched = rng.choice(["discrete", "linear", "cosine", "flow"])
    params = ["noise", "x_start", "flow"] if sched == "flow" else PARAMS
    steps = rng.randint(1, 12)
    return dict(sched=sched, param=rng.choice(params), cfg=rng.random() < 0.4, order=rng.randint(1, min(3, steps)),
                steps=steps, variant=rng.choice(["bh1", "bh2"]), alg=rng.choice(["dpmsolver++", "dpmsolver"]),
                corr=rng.random() < 0.75, lof=rng.random() < 0.5, d2z=rng.random() < 0.25,
                skip=rng.choice(["logSNR", "time_uniform", "time_quadratic"]))


def net64(x, t_in, c=None):
    """The test network, written once for torch fp32 tensors and fp64 numpy arrays."""
    k = 0.1 * x + 0.05 * np.sin(1e-3 * t_in) if isinstance(x, np.ndarray) else \
        0.1 * x + 0.05 * torch.sin(1e-3 * t_in).reshape(-1, *([1] * (x.dim() - 1)))
    return k if c is None else k + 0.03 * c


# (the runs start below T: at T, alpha_t is ~1e-3 on the cosine and flow schedules, and the x0 of a noise network,
# (x - sigma*eps)/alpha, carries fp32 cancellation of ~1e-4 relative into every later step)
T_START = 0.8


def run_product(c, calls, x):
    ns = schedule(c["sched"])

    def net(xx, tt, cc=None):
        calls.append((xx.clone(), tt.clone()))
        out = 0.1 * xx + 0.05 * torch.sin(1e-3 * tt).reshape(-1, 1, 1)
        return out if cc is None else out + 0.03 * cc.reshape(-1, 1, 1)

    kw = dict(model_type=c["param"])
    if c["cfg"]:
        B = x.shape[0]
        kw.update(guidance_type="classifier-free", condition=torch.ones(B), unconditional_condition=-torch.ones(B),
                  guidance_scale=2.5)
    s = UniPC(model_wrapper(net, ns, **kw), ns, algorithm_type=c["alg"], variant=c["variant"])
    return ns, s, s.sample(x, steps=c["steps"], t_start=T_START * ns.T, order=c["order"], skip_type=c["skip"],
                           lower_order_final=c["lof"],
                           use_corrector=c["corr"], denoise_to_zero=c["d2z"], return_intermediate=True)


def oracle64(c, ns, s, x):
    """The fp64 transcription on the product's fp32 grid and marginals, with the same network and conversions."""
    ts = s.get_time_steps(c["skip"], T_START * ns.T, 1. / ns.total_N, c["steps"], "cpu")
    marg = P.Marginals(ns, ts)
    lam, al, sg, ale = (v.double().numpy() for v in (marg.lam, marg.alpha, marg.sigma, marg.alpha_e))
    tin = model_wrapper(lambda *a: None, ns).get_model_input_time(ts).double().numpy()
    data = c["alg"] == "dpmsolver++"
    inputs = []

    def convert(o, xx, i):
        p = c["param"]
        if p == "flow":
            return xx - sg[i] * o if data else xx + ale[i] * o
        eps = {"noise": o, "x_start": (xx - ale[i] * o) / sg[i], "v": ale[i] * o + sg[i] * xx, "score": -sg[i] * o}[p]
        return (xx - sg[i] * eps) / ale[i] if data else eps

    def model(xx, i):
        inputs.append((xx, i))
        if not c["cfg"]:
            return convert(net64(xx, tin[i]), xx, i)
        tc, tu = convert(net64(xx, tin[i], 1.0), xx, i), convert(net64(xx, tin[i], -1.0), xx, i)
        return tu + 2.5 * (tc - tu)

    xN, xs = unipc_fp64(model, al, sg, lam, x.double().numpy(), c["order"], data, c["variant"] == "bh2", c["corr"],
                        c["lof"], return_intermediate=True)
    return xN, xs, inputs, tin


@pytest.mark.parametrize("seed", range(40))
def test_product_matches_the_fp64_transcription(uni_backend, seed):
    rng = random.Random(seed)
    c = draw(rng)
    x = torch.randn(2, 3, 4, generator=torch.Generator().manual_seed(seed))
    calls = []
    ns, s, (y, inter) = run_product(c, calls, x)
    xN, xs, inputs, tin = oracle64(c, ns, s, x)
    scale = max(1.0, float(np.abs(xN).max()))
    got = inter[c["steps"]]
    assert float(np.abs(got.double().numpy() - xN).max()) <= 1e-5 * scale, c
    for k in range(c["steps"] + 1):         # x_T, the corrected states, x_N
        assert float(np.abs(inter[k].double().numpy() - xs[k]).max()) <= 1e-5 * scale, (c, k)
    # the network calls: one per evaluation (+1 for denoise_to_zero), at the predictor outputs, with the right times
    n_eval = c["steps"] + (1 if c["d2z"] else 0)
    assert len(calls) == n_eval, c
    copies = 2 if c["cfg"] else 1
    for (xin, tt), (x64, i) in zip(calls, inputs):
        assert xin.shape[0] == copies * x.shape[0]
        assert float(np.abs(xin[:x.shape[0]].double().numpy() - x64).max()) <= 1e-5 * scale, (c, i)
        assert torch.equal(tt, torch.full_like(tt, float(np.float32(tin[i]))))
        if c["cfg"]:
            assert torch.equal(xin[:x.shape[0]], xin[x.shape[0]:])
    # launches: the LIN1 step plus one UniPC launch per later evaluation, conversion launches only where the
    # network's output is not the buffered value itself
    kinds = [e for e in uni_backend.log if e[0] == "unipc"]
    assert len(kinds) == c["steps"] - 1


def test_thresholding_adds_one_quantile_per_evaluation(uni_backend):
    ns = schedule("discrete")
    net = lambda x, t: 0.1 * x + 2.0
    s = UniPC(model_wrapper(net, ns), ns, correcting_x0_fn="dynamic_thresholding")
    s.sample(torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(1)), steps=6, order=3)
    log = uni_backend.log
    assert sum(e[0] == "quantile" for e in log) == 6
    assert sum(e[0] == "unipc" for e in log) == 5
    assert len(log) == 12          # 6 quantiles, the LIN1 step, 5 UniPC launches


# ---- 5. hooks, intermediates, inverse, rejected arguments ----------------------------------------------------------------

@pytest.mark.parametrize("sd", [None, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("order", [1, 2, 3])
def test_identity_xt_hook_is_bit_identical(uni_backend, sd, order):
    ns = schedule("discrete")
    net = lambda x, t: 0.1 * x + 0.05 * torch.sin(1e-3 * t).reshape(-1, 1, 1, 1)
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(3))
    seen = []

    def hook(xx, t, step):
        seen.append(step)
        return xx

    a = UniPC(model_wrapper(net, ns), ns, state_dtype=sd).sample(x, steps=8, order=order, return_intermediate=True)
    b = UniPC(model_wrapper(net, ns), ns, state_dtype=sd, correcting_xt_fn=hook).sample(
        x, steps=8, order=order, return_intermediate=True)
    assert torch.equal(a[0], b[0])
    assert all(torch.equal(u, v) for u, v in zip(a[1], b[1]))
    assert seen == list(range(9))


def test_intermediates_are_the_corrected_states(uni_backend):
    ns = schedule("linear")
    net = lambda x, t: 0.1 * x + 0.05 * torch.sin(t).reshape(-1, 1, 1)
    x = torch.randn(2, 3, 4, generator=torch.Generator().manual_seed(4))
    s = UniPC(model_wrapper(net, ns), ns)
    y, inter = s.sample(x, steps=6, order=2, return_intermediate=True)
    assert len(inter) == 7 and torch.equal(inter[0], x) and torch.equal(inter[-1], y)
    _, inter_nc = s.sample(x, steps=6, order=2, return_intermediate=True, use_corrector=False)
    assert not torch.equal(inter[2], inter_nc[2])        # the corrector moved x_2


def test_inverse_runs_the_reversed_time_range(uni_backend):
    ns = schedule("discrete")
    net = lambda x, t: 0.1 * x + 0.05 * torch.sin(1e-3 * t).reshape(-1, 1, 1, 1)
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(6))
    s = UniPC(model_wrapper(net, ns), ns)
    a = s.inverse(x, steps=5, order=2)
    b = s.sample(x, steps=5, order=2, t_start=1. / ns.total_N, t_end=ns.T)
    assert torch.equal(a, b) and torch.isfinite(a).all()


def test_rejections_launch_nothing(uni_backend):
    ns = schedule("discrete")
    net = lambda x, t, c=None: 0.1 * x
    x = torch.randn(2, 4, 8, 8)
    B = x.shape[0]
    with pytest.raises(ValueError):
        UniPC(model_wrapper(net, ns), ns, variant="bh3")
    cases = [
        (model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B), unconditional_condition=torch.zeros(B),
                       guidance_scale=torch.tensor([2., 3.])), {}),
        (model_wrapper(net, ns, guidance_type="classifier-free", condition=[torch.ones(B), torch.ones(B)],
                       unconditional_condition=torch.zeros(B), guidance_scale=[2., 3.]), {}),
        (model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B), unconditional_condition=torch.zeros(B),
                       guidance_scale=2., guidance_rescale=0.7), {}),
        (model_wrapper(net, ns), dict(order=4)),
        (model_wrapper(net, ns), dict(order=0)),
        (model_wrapper(net, ns), dict(order=3, steps=2)),
    ]
    for fn, kw in cases:
        s = UniPC(fn, ns)
        before = uni_backend.launch_count()
        with pytest.raises(ValueError):
            s.sample(x, **dict(dict(steps=5, order=2), **kw))
        assert uni_backend.launch_count() == before
    for attr in ("reference_rounding", "plan_broadcast"):
        s = UniPC(model_wrapper(net, ns), ns)
        setattr(s, attr, True)
        before = uni_backend.launch_count()
        with pytest.raises(ValueError):
            s.sample(x, steps=5)
        assert uni_backend.launch_count() == before


def test_exported_from_the_drop_in_module():
    import dpm_solver_pytorch
    assert dpm_solver_pytorch.UniPC is UniPC
