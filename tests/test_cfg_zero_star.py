"""CFG-Zero* (`model_wrapper(..., cfg_zero_star=True, cfg_zero_init_steps=K)`) on the CPU: the product's host logic on
the numpy executor (tests/cfgzero_oracle.py). s* against exactly rounded sums; sample() bit for bit against the
UNMODIFIED reference solver driving a plain network that returns the CFG-Zero* output (zeros for its first K calls);
UniPC; per-sample rows, the scale-1 bypass, batch sharding and the rejections."""
import os

import numpy as np
import pytest
import torch

from cases import make_betas
from cfgzero_oracle import CFGZeroOracle, guided_net, s_star_exact, s_star_fsum
from oracle import ref_loader

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
B, SHAPE = 2, (2, 3, 6, 6)
W = 4.5
MODEL_TYPES = ["noise", "x_start", "v", "score", "flow", "edm"]


@pytest.fixture()
def cfz_backend():
    from dpm_solver_b200 import ops
    be = CFGZeroOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def net(x, t, c):
    """A time-independent network whose two halves differ nonlinearly (u is far from a multiple of c)."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x + 0.25 * cc * torch.cos(0.7 * x) - 0.1


def counted(calls):
    def f(x, t, c):
        calls.append(tuple(x.shape))
        return net(x, t, c)
    return f


def product_schedule(mt):
    import dpm_solver_b200 as new
    if mt == "flow":
        return new.NoiseScheduleFlow(shift=3.0)
    if mt == "edm":
        return new.NoiseScheduleEDM()
    return new.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def reference_schedule(mt):
    if mt == "flow":
        from flow_oracle import reference_schedule as flow
        return flow(3.0)
    if mt == "edm":
        from edm_oracle import reference_schedule as edm
        return edm()
    ref = ref_loader.load("dpm_solver_pytorch")
    return ref.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def wrap(mt, ns, w=W, model=net, **kw):
    import dpm_solver_b200 as new
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free", condition=torch.ones(B, 1),
                             unconditional_condition=torch.zeros(B, 1), guidance_scale=w, **kw)


def reference(mt, algo, w, K=0, thr=False, calls=None):
    """The unmodified reference solver driven by guidance_type="uncond" on the CFG-Zero* network."""
    ref = ref_loader.load("dpm_solver_pytorch")
    rns = reference_schedule(mt)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), w, K, calls)
    if mt == "flow":
        from flow_oracle import reference_solver
        return reference_solver(g, rns, algo, thresholding=thr)
    if mt == "edm":
        from edm_oracle import reference_solver
        return reference_solver(g, rns, algo, thresholding=thr)
    return ref.DPM_Solver(ref.model_wrapper(g, rns, model_type=mt), rns, algorithm_type=algo,
                          correcting_x0_fn="dynamic_thresholding" if thr else None)


def x_T(seed=0):
    return torch.randn(SHAPE, generator=torch.Generator().manual_seed(seed))


# ---- s* --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("per_sample", [7, 8, 9, 8192 + 16, 8193, 3 * 64 * 64])
def test_s_star_within_one_ulp_of_fsum(per_sample):
    rng = np.random.default_rng(per_sample)
    c = rng.standard_normal((3, per_sample)).astype(np.float32)
    u = (0.7 * c + 0.5 * rng.standard_normal((3, per_sample))).astype(np.float32)
    u[2] *= np.float32(1e-3)            # a small unconditional output: the 1e-8 is still negligible
    got, want = s_star_exact(c, u), s_star_fsum(c, u)
    ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    assert ulps.max() <= 1, (got, want)
    # u = 0: s* = 0 / 1e-8 = 0
    assert s_star_exact(c[:1], np.zeros_like(c[:1]))[0] == 0.0


def test_s_star_reads_each_sample_alone():
    rng = np.random.default_rng(1)
    c = rng.standard_normal((4, 8193)).astype(np.float32)
    u = rng.standard_normal((4, 8193)).astype(np.float32)
    full = s_star_exact(c, u)
    for b in range(4):
        assert s_star_exact(c[b:b + 1], u[b:b + 1])[0] == full[b]


# ---- sample() against the reference ----------------------------------------------------------------------------------

METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2),
           ("singlestep", 3), ("adaptive", 2)]
# (scale, thresholding, zero-init steps)
CONFIGS = [(W, False, 0), (W, True, 0), ("per_sample", False, 0), (W, False, 2), ("per_sample", True, 1)]


@needs_ref
@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("method,order", METHODS)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
def test_sample_matches_reference(cfz_backend, mt, method, order, algo, cfg, capsys):
    import dpm_solver_b200 as new
    w, thr, K = CONFIGS[cfg]
    if method == "adaptive" and K:
        pytest.skip("zero-init is refused with the adaptive solver (test_rejections_launch_nothing)")
    if thr and algo == "dpmsolver":
        pytest.skip("thresholding acts on the data prediction")
    w = torch.tensor([1.0, 3.0]) if w == "per_sample" else w
    ns = product_schedule(mt)
    calls, ref_calls = [], []
    fn = wrap(mt, ns, w, model=counted(calls), cfg_zero_star=True, cfg_zero_init_steps=K)
    skw = dict(steps=6, order=order, method=method)
    if method == "adaptive":
        skw = dict(order=order, method=method, atol=0.05, rtol=0.1)
    y = new.DPM_Solver(fn, ns, algorithm_type=algo,
                       correcting_x0_fn="dynamic_thresholding" if thr else None).sample(x_T(), **skw)
    yr = reference(mt, algo, w, K, thr, ref_calls).sample(x_T(), **skw)
    capsys.readouterr()
    assert len(calls) == len(ref_calls) and all(c == (2 * B,) + SHAPE[1:] for c in calls)
    if method == "adaptive":
        # the host controller's step-size scalars are the reference's to within an fp32 rounding, as for plain CFG
        # (tests/test_cfg_per_sample.py): the same evaluations, the result within 1e-5
        err = float((y.double() - yr.double()).abs().max() / yr.double().abs().max())
        assert err <= 1e-5, err
        return
    assert torch.equal(y, yr), float((y - yr).abs().max())
    if K:
        calls0 = []
        new.DPM_Solver(wrap(mt, ns, w, model=counted(calls0), cfg_zero_star=True), ns, algorithm_type=algo,
                       correcting_x0_fn="dynamic_thresholding" if thr else None).sample(x_T(), **skw)
        assert len(calls0) - len(calls) == K


@needs_ref
@pytest.mark.parametrize("mt", ["noise", "flow", "edm"])
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_zero_init_counts_singlestep_evaluations(cfz_backend, mt, K):
    """Singlestep order 3: every intermediate evaluation counts, so K = 2 zeroes two of the first step's three."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    calls, ref_calls = [], []
    skw = dict(steps=6, order=3, method="singlestep")
    y = new.DPM_Solver(wrap(mt, ns, model=counted(calls), cfg_zero_star=True, cfg_zero_init_steps=K), ns).sample(
        x_T(), **skw)
    yr = reference(mt, "dpmsolver++", W, K, calls=ref_calls).sample(x_T(), **skw)
    assert torch.equal(y, yr)
    assert len(calls) == 6 - K == len(ref_calls)


@needs_ref
@pytest.mark.parametrize("mt", ["noise", "v", "flow", "edm"])
@pytest.mark.parametrize("K", [5, 6, 7])
def test_zero_init_counts_denoise_to_zero(cfz_backend, mt, K):
    """Multistep with 6 steps evaluates 6 times, then denoise_to_zero once more: K = 7 zeroes that one too."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    calls = []
    skw = dict(steps=6, order=2, method="multistep", denoise_to_zero=True)
    y = new.DPM_Solver(wrap(mt, ns, model=counted(calls), cfg_zero_star=True, cfg_zero_init_steps=K), ns).sample(
        x_T(), **skw)
    yr = reference(mt, "dpmsolver++", W, K).sample(x_T(), **skw)
    assert torch.equal(y, yr)
    assert len(calls) == 7 - K


def test_zero_init_flow_x0_is_the_state(cfz_backend):
    """A zero-init evaluation of a flow network is x0 = x exactly, and the network is not called."""
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    calls = []
    s = new.DPM_Solver(wrap("flow", ns, model=counted(calls), cfg_zero_star=True, cfg_zero_init_steps=1), ns)
    x = x_T(4)
    with s._apg_scope():
        x0 = s.data_prediction_fn(x, torch.tensor([0.7]))
        assert torch.equal(x0, x) and calls == []
        s.data_prediction_fn(x, torch.tensor([0.7]))
        assert len(calls) == 1
    # outside a run: never zeroed
    assert not torch.equal(s.data_prediction_fn(x, torch.tensor([0.7])), x)


# ---- UniPC -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("K,thr", [(0, False), (2, False), (1, True)])
def test_unipc_matches_the_guided_network(cfz_backend, mt, algo, K, thr):
    """UniPC hands the materialised fp32 g to its launch as one network output: bit for bit the run on a network that
    returns g."""
    import dpm_solver_b200 as new
    if thr and algo == "dpmsolver":
        pytest.skip("thresholding acts on the data prediction")
    ns = product_schedule(mt)
    kw = dict(algorithm_type=algo, variant="bh2", correcting_x0_fn="dynamic_thresholding" if thr else None)
    calls = []
    y = new.UniPC(wrap(mt, ns, model=counted(calls), cfg_zero_star=True, cfg_zero_init_steps=K), ns, **kw).sample(
        x_T(), steps=6, order=3)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), W, K)
    yg = new.UniPC(new.model_wrapper(lambda x, t: g(x, t), ns, model_type=mt), ns, **kw).sample(
        x_T(), steps=6, order=3)
    assert torch.equal(y, yg)
    assert len(calls) == 6 - K


@pytest.mark.parametrize("mt", ["noise", "flow"])
def test_unipc_vs_fp64_transcription(cfz_backend, mt):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import plan as P
    from unipc_oracle import unipc_fp64
    ns = product_schedule(mt)
    s = new.UniPC(wrap(mt, ns, cfg_zero_star=True, cfg_zero_init_steps=1), ns)
    y = s.sample(x_T(), steps=8, order=2)
    ts = s.get_time_steps("time_uniform", ns.T, 1. / ns.total_N, 8, "cpu")
    marg = P.Marginals(ns, ts)
    lam, al, sg, ale = (v.double().numpy() for v in (marg.lam, marg.alpha, marg.sigma, marg.alpha_e))
    n = {"k": 0}

    def model(xx, i):
        n["k"] += 1
        xt = torch.from_numpy(xx)
        out_u, out_c = net(torch.cat([xt, xt]), None, torch.cat([torch.zeros(B, 1), torch.ones(B, 1)])).chunk(2)
        cu, uu = out_c.numpy(), out_u.numpy()
        sv = ((cu * uu).reshape(B, -1).sum(1) / ((uu * uu).reshape(B, -1).sum(1) + 1e-8)).reshape(-1, 1, 1, 1)
        g = 0 * cu if n["k"] == 1 else sv * uu + W * (cu - sv * uu)
        return xx - sg[i] * g if mt == "flow" else (xx - sg[i] * g) / ale[i]
    xN = unipc_fp64(model, al, sg, lam, x_T().double().numpy(), 2, True, True, True, True)
    assert float(np.abs(y.double().numpy() - xN).max()) <= 1e-4 * max(1.0, float(np.abs(xN).max()))


def test_unipc_launches(cfz_backend):
    """UniPC: per guided evaluation the s* pass and one FORM_NONE launch that materialises g; the zero-init evaluation
    is a launch on the zero output alone."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    new.UniPC(wrap("noise", ns, cfg_zero_star=True, cfg_zero_init_steps=1), ns).sample(x_T(), steps=5, order=2)
    assert sum(e[0] == "cfgzero_scale" for e in cfz_backend.log) == 4
    assert sum(1 for e in cfz_backend.log if e[0] == 0 and e[1] == 2) == 4
    assert sum(1 for e in cfz_backend.log if e[0] == "unipc" and e[1] == 1) == 4


# ---- rows, bypass, direct calls, sharding ----------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_per_sample_rows_equal_their_scalar_runs(cfz_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    kw = dict(steps=5, order=2)
    ws = [1.0, 3.0]
    yb = new.DPM_Solver(wrap(mt, ns, w=torch.tensor(ws), cfg_zero_star=True, cfg_zero_init_steps=1), ns).sample(
        x_T(), **kw)
    for b, w in enumerate(ws):
        yw = new.DPM_Solver(wrap(mt, ns, w=w, cfg_zero_star=True, cfg_zero_init_steps=1), ns).sample(x_T(), **kw)
        assert torch.equal(yb[b:b + 1], yw[b:b + 1])
    # a scale-1 row is the conditional output alone: the plain run's row
    y0 = new.DPM_Solver(wrap(mt, ns, w=1.0), ns).sample(x_T(), **kw)
    y1 = new.DPM_Solver(wrap(mt, ns, w=torch.tensor(ws), cfg_zero_star=True), ns).sample(x_T(), **kw)
    assert torch.equal(y1[:1], y0[:1]) and not torch.equal(y1[1:], y0[1:])


@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_scalar_scale_one_keeps_the_bypass(cfz_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    calls = []
    cfz_backend.log.clear()
    y1 = new.DPM_Solver(wrap(mt, ns, w=1.0, model=counted(calls), cfg_zero_star=True), ns).sample(x_T(), steps=5)
    log1 = list(cfz_backend.log)
    cfz_backend.log.clear()
    y0 = new.DPM_Solver(wrap(mt, ns, w=1.0), ns).sample(x_T(), steps=5)
    assert torch.equal(y0, y1) and log1 == cfz_backend.log
    assert all(c[0] == B for c in calls)


@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_direct_model_fn_call(cfz_backend, mt):
    """model_fn(x, t) returns the guided raw output g converted to noise, and is never zeroed."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    fn = wrap(mt, ns, cfg_zero_star=True, cfg_zero_init_steps=3)
    x, t = x_T(3), torch.full((B,), 0.5)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), W)
    want = new.model_wrapper(lambda xx, tt: g(xx, tt), ns, model_type=mt)(x, t)
    assert torch.equal(fn(x, t), want)


def test_two_sample_calls_and_a_fresh_solver_are_bit_identical(cfz_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    fn = wrap("flow", ns, cfg_zero_star=True, cfg_zero_init_steps=2)
    s = new.DPM_Solver(fn, ns)
    y1, y2 = s.sample(x_T(), steps=5, order=2), s.sample(x_T(), steps=5, order=2)
    y3 = new.DPM_Solver(fn, ns).sample(x_T(), steps=5, order=2)
    assert torch.equal(y1, y2) and torch.equal(y1, y3)


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dpm_solver_b200 import ops
        import dpm_solver_b200 as new
        ops.set_backend(CFGZeroOracle())
        ns = product_schedule("flow")
        x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))[2 * rank:2 * rank + 2]
        fn = wrap("flow", ns, w=torch.tensor([3.0, 1.0, 5.0, 2.0])[2 * rank:2 * rank + 2], cfg_zero_star=True,
                  cfg_zero_init_steps=1)
        y = new.DPM_Solver(fn, ns, plan_broadcast=True).sample(x, steps=5, order=2)
        q.put((rank, y))
    finally:
        dist.destroy_process_group()


def test_batch_sharding_needs_no_collective(cfz_backend):
    """Two gloo ranks of two samples each equal the unsharded run of four: s* is per sample."""
    import socket
    import torch.multiprocessing as mp
    import dpm_solver_b200 as new
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    ns = product_schedule("flow")
    x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))
    fn = new.model_wrapper(net, ns, model_type="flow", guidance_type="classifier-free", condition=torch.ones(4, 1),
                           unconditional_condition=torch.zeros(4, 1), guidance_scale=torch.tensor([3.0, 1.0, 5.0, 2.0]),
                           cfg_zero_star=True, cfg_zero_init_steps=1)
    y = new.DPM_Solver(fn, ns).sample(x, steps=5, order=2)
    assert torch.equal(torch.cat([got[0], got[1]]), y)


# ---- rejections ------------------------------------------------------------------------------------------------------

def _rejections():
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    uc, c = torch.zeros(B, 1), torch.ones(B, 1)
    base = dict(guidance_type="classifier-free", condition=c, unconditional_condition=uc, guidance_scale=W)
    bad_wrap = [
        dict(base, condition=[c, c], guidance_scale=[2.0, 3.0], cfg_zero_star=True),
        dict(base, guidance_rescale=0.7, cfg_zero_star=True),
        dict(base, apg_eta=0.0, cfg_zero_star=True),
        dict(guidance_type="uncond", cfg_zero_star=True),
        dict(guidance_type="classifier", classifier_fn=lambda *a: None, condition=c, cfg_zero_star=True),
        dict(base, unconditional_condition=None, cfg_zero_star=True),
        dict(base, cfg_zero_star=True, cfg_zero_init_steps=-1),
        dict(base, cfg_zero_star=True, cfg_zero_init_steps=1.0),
        dict(base, cfg_zero_star=True, cfg_zero_init_steps=True),
        dict(base, cfg_zero_init_steps=1),
    ]
    for kw in bad_wrap:
        yield lambda kw=kw: new.model_wrapper(net, ns, **kw)
    fn = new.model_wrapper(net, ns, cfg_zero_star=True, **base)
    yield lambda: new.DPM_Solver(fn, ns, reference_rounding=True)
    fz = new.model_wrapper(net, ns, cfg_zero_star=True, cfg_zero_init_steps=1, **base)
    yield lambda: new.DPM_Solver(fz, ns).sample(x_T(), order=2, method="adaptive")
    yield lambda: new.DPM_Solver(fz, ns).inverse(x_T(), order=2, method="adaptive")


def test_rejections_launch_nothing(cfz_backend):
    n = 0
    for call in _rejections():
        before = cfz_backend.launch_count()
        with pytest.raises(ValueError):
            call()
        assert cfz_backend.launch_count() == before
        n += 1
    assert n == 13


def test_adaptive_without_zero_init_runs(cfz_backend, capsys):
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    y = new.DPM_Solver(wrap("flow", ns, cfg_zero_star=True), ns).sample(x_T(), order=2, method="adaptive",
                                                                         atol=0.05, rtol=0.1)
    capsys.readouterr()
    assert torch.isfinite(y).all()
