"""TCFG (`model_wrapper(..., tcfg=True)`) on the CPU: the product's host logic on the numpy executor
(tests/tcfg_oracle.py). The closed-form words against a float64 SVD transcription of diffusers' guider and against
exactly rounded sums; sample() bit for bit against the UNMODIFIED reference solver driving a plain network that
returns the TCFG output; UniPC; the condition-blind identity, per-sample rows, the scale-1 bypass, direct calls, launch
counts, batch sharding and the rejections."""
import os

import numpy as np
import pytest
import torch

from cases import make_betas
from oracle import ref_loader
from tcfg_oracle import (NAN32, TCFGOracle, guided_net, tcfg_svd_reference, words_closed_form, words_exact,
                         words_fsum)

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
B, SHAPE = 2, (2, 3, 6, 6)
W = 4.5
MODEL_TYPES = ["noise", "x_start", "v", "score", "flow", "edm"]


@pytest.fixture()
def tcfg_backend():
    from dpm_solver_b200 import ops
    be = TCFGOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def net(x, t, c):
    """A time-independent network whose two halves differ nonlinearly (u is far from a multiple of c)."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x + 0.25 * cc * torch.cos(0.7 * x) - 0.1


def blind(x, t, c):
    """A network that ignores the condition: c == u."""
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x - 0.1


def counted(calls, model=net):
    def f(x, t, c):
        calls.append(tuple(x.shape))
        return model(x, t, c)
    return f


def product_schedule(mt, kind="discrete"):
    import dpm_solver_b200 as new
    if mt == "flow":
        return new.NoiseScheduleFlow(shift=3.0)
    if mt == "edm":
        return new.NoiseScheduleEDM()
    if kind != "discrete":
        return new.NoiseScheduleVP(kind)
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


def reference(mt, algo, w, thr=False, calls=None):
    """The unmodified reference solver driven by guidance_type="uncond" on the TCFG network."""
    ref = ref_loader.load("dpm_solver_pytorch")
    rns = reference_schedule(mt)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), w, calls)
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


def ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


# ---- the words -------------------------------------------------------------------------------------------------------

def _pairs(seed, n=200):
    """Seeded non-degenerate (c, u) pairs of varied size, angle and norm ratio."""
    rng = np.random.default_rng(seed)
    for k in range(n):
        D = int(rng.integers(2, 300))
        c = rng.standard_normal(D) * 10.0 ** rng.uniform(-2, 2)
        mix = rng.uniform(-1, 1)
        u = mix * c + rng.standard_normal(D) * 10.0 ** rng.uniform(-2, 2)
        yield c, u


def test_closed_form_matches_the_svd_transcription():
    """u' = wu*u + wc*c from the fp64 closed form, before any fp32 rounding, within 1e-12 of diffusers' SVD form."""
    worst = 0.0
    for c, u in _pairs(7):
        A, Bs, C = float(u @ u), float(u @ c), float(c @ c)
        h = 0.5 * (A - C)
        r = np.sqrt(h * h + Bs * Bs)
        p, q = (Bs, (-h) + r) if C >= A else (h + r, Bs)
        n2 = p * p + q * q
        up = (p * p / n2) * u + (p * q / n2) * c
        _, want = tcfg_svd_reference(c[None], u[None], W)
        worst = max(worst, float(np.abs(up - want[0]).max() / np.abs(want[0]).max()))
    assert worst <= 1e-12, worst


@pytest.mark.parametrize("per_sample", [7, 8, 9, 8192 + 16, 8193, 3 * 64 * 64])
def test_executor_words_within_two_ulp_of_fsum(per_sample):
    rng = np.random.default_rng(per_sample)
    c = rng.standard_normal((3, per_sample)).astype(np.float32)
    u = (0.7 * c + 0.5 * rng.standard_normal((3, per_sample))).astype(np.float32)
    u[2] *= np.float32(1e-3)
    got, want = words_exact(c, u), words_fsum(c, u)
    assert ulps(got, want).max() <= 2, (got, want)


def test_words_read_each_sample_alone():
    rng = np.random.default_rng(1)
    c = rng.standard_normal((4, 8193)).astype(np.float32)
    u = rng.standard_normal((4, 8193)).astype(np.float32)
    full = words_exact(c, u)
    for b in range(4):
        assert np.array_equal(words_exact(c[b:b + 1], u[b:b + 1])[0], full[b])


def test_constructed_words():
    rng = np.random.default_rng(3)
    D = 64
    v = rng.standard_normal(D).astype(np.float32)
    # c == u: exactly (0.5, 0.5)
    assert words_exact(v[None], v[None]).tolist() == [[0.5, 0.5]]
    # c _|_ u with equal norms, and both zero: (1, 0)
    e1, e2 = np.zeros(D, np.float32), np.zeros(D, np.float32)
    e1[0], e2[1] = 3.0, 3.0
    assert words_exact(e1[None], e2[None]).tolist() == [[1.0, 0.0]]
    z = np.zeros((1, D), np.float32)
    assert words_exact(z, z).tolist() == [[1.0, 0.0]]
    # c _|_ u with ||c|| > ||u||: u' = 0, (0, 0)
    e2[1] = 2.0
    assert words_exact(e1[None], e2[None]).tolist() == [[0.0, 0.0]]
    # ... and with ||u|| > ||c||: u' = u, (1, 0)
    assert words_exact(e2[None], e1[None]).tolist() == [[1.0, 0.0]]
    # an inf or NaN output: NaN words, with the device's NaN
    for bad in (np.inf, -np.inf, np.nan):
        cb = v.copy()
        cb[5] = bad
        for cc, uu in ((cb, v), (v, cb)):
            w = words_exact(cc[None], uu[None])
            assert np.isnan(w).all() and (w.view(np.uint32) == NAN32.view(np.uint32)).all()
    # rank 1 (c = k*u, here k = 2): u' = wu*u + wc*k*u = u in exact arithmetic, so wu + k*wc = 1
    wu, wc = words_closed_form(4.0, 8.0, 16.0)[0].astype(np.float64)
    assert abs(wu + 2.0 * wc - 1.0) <= 1e-7
    wu, wc = words_exact(2 * v[None], v[None])[0].astype(np.float64)
    assert abs(wu + 2.0 * wc - 1.0) <= 1e-6


# ---- sample() against the reference ----------------------------------------------------------------------------------

METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2),
           ("singlestep", 3), ("singlestep_fixed", 2), ("adaptive", 2)]
CONFIGS = [(W, False), (W, True), ("per_sample", False), ("per_sample", True)]


@needs_ref
@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("method,order", METHODS)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
def test_sample_matches_reference(tcfg_backend, mt, method, order, algo, cfg, capsys):
    import dpm_solver_b200 as new
    w, thr = CONFIGS[cfg]
    if thr and algo == "dpmsolver":
        pytest.skip("thresholding acts on the data prediction")
    w = torch.tensor([1.0, 3.0]) if w == "per_sample" else w
    ns = product_schedule(mt)
    calls, ref_calls = [], []
    fn = wrap(mt, ns, w, model=counted(calls), tcfg=True)
    skw = dict(steps=6, order=order, method=method)
    if method == "adaptive":
        skw = dict(order=order, method=method, atol=0.05, rtol=0.1)
    y = new.DPM_Solver(fn, ns, algorithm_type=algo,
                       correcting_x0_fn="dynamic_thresholding" if thr else None).sample(x_T(), **skw)
    yr = reference(mt, algo, w, thr, ref_calls).sample(x_T(), **skw)
    capsys.readouterr()
    assert len(calls) == len(ref_calls) and all(c == (2 * B,) + SHAPE[1:] for c in calls)
    if method == "adaptive":
        # the host controller's step-size scalars are the reference's to within an fp32 rounding, as for plain CFG: the
        # same evaluations, the result within 1e-5
        err = float((y.double() - yr.double()).abs().max() / yr.double().abs().max())
        assert err <= 1e-5, err
        return
    assert torch.equal(y, yr), float((y - yr).abs().max())


@needs_ref
@pytest.mark.parametrize("mt", ["noise", "v", "flow", "edm"])
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
def test_denoise_to_zero_and_inverse_match_reference(tcfg_backend, mt, algo):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    skw = dict(steps=6, order=2, method="multistep", denoise_to_zero=True)
    y = new.DPM_Solver(wrap(mt, ns, tcfg=True), ns, algorithm_type=algo).sample(x_T(), **skw)
    yr = reference(mt, algo, W).sample(x_T(), **skw)
    assert torch.equal(y, yr)
    ikw = dict(steps=5, order=2, method="multistep")
    yi = new.DPM_Solver(wrap(mt, ns, tcfg=True), ns, algorithm_type=algo).inverse(x_T(1), **ikw)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), W)
    yg = new.DPM_Solver(new.model_wrapper(lambda x, t: g(x, t), ns, model_type=mt), ns,
                        algorithm_type=algo).inverse(x_T(1), **ikw)
    assert torch.equal(yi, yg)


@pytest.mark.parametrize("kind", ["linear", "cosine"])
def test_continuous_vp_schedules(tcfg_backend, kind):
    import dpm_solver_b200 as new
    ns = product_schedule("noise", kind)
    y = new.DPM_Solver(wrap("noise", ns, tcfg=True), ns).sample(x_T(), steps=5, order=2)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), W)
    yg = new.DPM_Solver(new.model_wrapper(lambda x, t: g(x, t), ns), ns).sample(x_T(), steps=5, order=2)
    assert torch.equal(y, yg)


# ---- UniPC -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("thr", [False, True])
def test_unipc_matches_the_guided_network(tcfg_backend, mt, algo, thr):
    """UniPC hands the materialised fp32 g to its launch as one network output: bit for bit the run on a network that
    returns g."""
    import dpm_solver_b200 as new
    if thr and algo == "dpmsolver":
        pytest.skip("thresholding acts on the data prediction")
    ns = product_schedule(mt)
    kw = dict(algorithm_type=algo, variant="bh2", correcting_x0_fn="dynamic_thresholding" if thr else None)
    calls = []
    y = new.UniPC(wrap(mt, ns, model=counted(calls), tcfg=True), ns, **kw).sample(x_T(), steps=6, order=3)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), W)
    yg = new.UniPC(new.model_wrapper(lambda x, t: g(x, t), ns, model_type=mt), ns, **kw).sample(
        x_T(), steps=6, order=3)
    assert torch.equal(y, yg)
    assert len(calls) == 6


# ---- identities, rows, bypass, direct calls, counts, sharding ----------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("state_dtype", [None, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("w", [W, 0.0, "per_sample"])
def test_condition_blind_run_equals_the_unguided_run(tcfg_backend, mt, state_dtype, w):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    w = torch.tensor([2.0, 7.5]) if w == "per_sample" else w
    kw = dict(steps=6, order=2)
    y = new.DPM_Solver(wrap(mt, ns, w, model=blind, tcfg=True), ns, state_dtype=state_dtype).sample(x_T(), **kw)
    y0 = new.DPM_Solver(new.model_wrapper(lambda x, t: blind(x, t, None), ns, model_type=mt), ns,
                        state_dtype=state_dtype).sample(x_T(), **kw)
    assert torch.equal(y, y0)


@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_per_sample_rows_equal_their_scalar_runs(tcfg_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    kw = dict(steps=5, order=2)
    ws = [2.0, 6.0]
    yb = new.DPM_Solver(wrap(mt, ns, w=torch.tensor(ws), tcfg=True), ns).sample(x_T(), **kw)
    for b, w in enumerate(ws):
        yw = new.DPM_Solver(wrap(mt, ns, w=w, tcfg=True), ns).sample(x_T(), **kw)
        assert torch.equal(yb[b:b + 1], yw[b:b + 1])
    # a scale-1 row is the conditional output alone: the plain run's row
    y0 = new.DPM_Solver(wrap(mt, ns, w=1.0), ns).sample(x_T(), **kw)
    y1 = new.DPM_Solver(wrap(mt, ns, w=torch.tensor([1.0, 3.0]), tcfg=True), ns).sample(x_T(), **kw)
    assert torch.equal(y1[:1], y0[:1]) and not torch.equal(y1[1:], y0[1:])


@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_scalar_scale_one_keeps_the_bypass(tcfg_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    calls = []
    tcfg_backend.log.clear()
    y1 = new.DPM_Solver(wrap(mt, ns, w=1.0, model=counted(calls), tcfg=True), ns).sample(x_T(), steps=5)
    log1 = list(tcfg_backend.log)
    tcfg_backend.log.clear()
    y0 = new.DPM_Solver(wrap(mt, ns, w=1.0), ns).sample(x_T(), steps=5)
    assert torch.equal(y0, y1) and log1 == tcfg_backend.log
    assert calls and all(c[0] == B for c in calls)


@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_direct_model_fn_call(tcfg_backend, mt):
    """model_fn(x, t) returns the guided raw output g converted to noise."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    fn = wrap(mt, ns, tcfg=True)
    x, t = x_T(3), torch.full((B,), 0.5)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), W)
    want = new.model_wrapper(lambda xx, tt: g(xx, tt), ns, model_type=mt)(x, t)
    assert torch.equal(fn(x, t), want)
    # per-sample time labels: one conversion per row, the words over the whole batch
    t2 = torch.tensor([0.5, 0.3])
    assert torch.equal(fn(x, t2), new.model_wrapper(lambda xx, tt: g(xx, tt), ns, model_type=mt)(x, t2))


def test_launch_and_network_call_counts(tcfg_backend):
    """Per guided evaluation: one network call on 2B rows, the words pass (2 launches) and the fused step; with
    thresholding one more launch materialises g."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    for thr, per_eval in ((False, 3), (True, 3 + 1)):
        calls = []
        s = new.DPM_Solver(wrap("noise", ns, model=counted(calls), tcfg=True), ns,
                           correcting_x0_fn="dynamic_thresholding" if thr else None)
        s0 = new.DPM_Solver(wrap("noise", ns), ns, correcting_x0_fn="dynamic_thresholding" if thr else None)
        tcfg_backend.log.clear()
        n0 = tcfg_backend.launch_count()
        s0.sample(x_T(), steps=5, order=2)
        plain = tcfg_backend.launch_count() - n0
        n0 = tcfg_backend.launch_count()
        s.sample(x_T(), steps=5, order=2)
        got = tcfg_backend.launch_count() - n0
        assert len(calls) == 5 and all(c == (2 * B,) + SHAPE[1:] for c in calls)
        assert sum(e[0] == "tcfg_words" for e in tcfg_backend.log) == 5
        assert got - plain == 5 * (per_eval - 1), (got, plain)


def test_two_sample_calls_and_a_fresh_solver_are_bit_identical(tcfg_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    fn = wrap("flow", ns, tcfg=True)
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
        ops.set_backend(TCFGOracle())
        ns = product_schedule("flow")
        x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))[2 * rank:2 * rank + 2]
        fn = wrap("flow", ns, w=torch.tensor([3.0, 1.0, 5.0, 2.0])[2 * rank:2 * rank + 2], tcfg=True)
        y = new.DPM_Solver(fn, ns, plan_broadcast=True).sample(x, steps=5, order=2)
        q.put((rank, y))
    finally:
        dist.destroy_process_group()


def test_batch_sharding_needs_no_collective(tcfg_backend):
    """Two gloo ranks of two samples each equal the unsharded run of four: the words are per sample."""
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
                           tcfg=True)
    y = new.DPM_Solver(fn, ns).sample(x, steps=5, order=2)
    assert torch.equal(torch.cat([got[0], got[1]]), y)


# ---- rejections ------------------------------------------------------------------------------------------------------

def _rejections(calls):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    uc, c = torch.zeros(B, 1), torch.ones(B, 1)
    model = counted(calls)
    base = dict(guidance_type="classifier-free", condition=c, unconditional_condition=uc, guidance_scale=W)
    bad_wrap = [
        dict(base, tcfg=1),
        dict(base, tcfg="yes"),
        dict(guidance_type="uncond", tcfg=True),
        dict(guidance_type="classifier", classifier_fn=lambda *a: None, condition=c, tcfg=True),
        dict(base, unconditional_condition=None, tcfg=True),
        dict(base, condition=[c, c], guidance_scale=[2.0, 3.0], tcfg=True),
        dict(base, guidance_mask=torch.ones(6, 6), tcfg=True),
        dict(base, guidance_rescale=0.7, tcfg=True),
        dict(base, apg_eta=0.0, tcfg=True),
        dict(base, cfg_zero_star=True, tcfg=True),
        dict(base, cfg_pp=True, tcfg=True),
    ]
    for kw in bad_wrap:
        yield lambda kw=kw: new.model_wrapper(model, ns, **kw)
    fn = new.model_wrapper(model, ns, tcfg=True, **base)
    yield lambda: new.DPM_Solver(fn, ns, reference_rounding=True)


def test_rejections_launch_nothing(tcfg_backend):
    n, calls = 0, []
    for call in _rejections(calls):
        before = tcfg_backend.launch_count()
        with pytest.raises(ValueError):
            call()
        assert tcfg_backend.launch_count() == before and calls == []
        n += 1
    assert n == 12
