"""Frequency-decoupled guidance (`model_wrapper(..., fdg_scales=[w_0, ..., w_{N-1}])`) on the CPU: the product's host
logic on the numpy executor (tests/fdg_oracle.py). The correction form against diffusers' per-level form; the
identities of the contract; sample() bit for bit against the UNMODIFIED reference solver driving a plain network that
returns the FDG output; UniPC, the adaptive solver, per-sample rows, shapes, direct calls, launch counts, batch sharding
and the rejections."""
import os

import numpy as np
import pytest
import torch

from cases import make_betas
from fdg_oracle import FDGOracle, down2, fdg_exact, fdg_fp64, guided_net, up2
from oracle import ref_loader

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
B, SHAPE = 2, (2, 3, 12, 16)
SCALES = [7.0, 3.5, 1.5]
MODEL_TYPES = ["noise", "x_start", "v", "score", "flow", "edm"]


@pytest.fixture()
def fdg_backend():
    from dpm_solver_b200 import ops
    be = FDGOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def net(x, t, c):
    """A time-independent network whose two halves differ in fine and coarse structure alike."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x + 0.25 * cc * torch.cos(0.7 * x + 0.3) - 0.1


def blind(x, t, c):
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


def wrap(mt, ns, scales=SCALES, model=net, b=B, **kw):
    import dpm_solver_b200 as new
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free", condition=torch.ones(b, 1),
                             unconditional_condition=torch.zeros(b, 1), fdg_scales=scales, **kw)


def guided_wrap(mt, ns, scales=SCALES, model=net, b=B):
    """The product's own uncond wrapper on a network that returns the FDG output."""
    import dpm_solver_b200 as new
    g = guided_net(model, torch.zeros(b, 1), torch.ones(b, 1), scales)
    return new.model_wrapper(lambda x, t: g(x, t), ns, model_type=mt)


def reference(mt, algo, scales, thr=False, calls=None):
    """The unmodified reference solver driven by guidance_type="uncond" on the FDG network."""
    ref = ref_loader.load("dpm_solver_pytorch")
    rns = reference_schedule(mt)
    g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), scales, calls)
    if mt == "flow":
        from flow_oracle import reference_solver
        return reference_solver(g, rns, algo, thresholding=thr)
    if mt == "edm":
        from edm_oracle import reference_solver
        return reference_solver(g, rns, algo, thresholding=thr)
    return ref.DPM_Solver(ref.model_wrapper(g, rns, model_type=mt), rns, algorithm_type=algo,
                          correcting_x0_fn="dynamic_thresholding" if thr else None)


def x_T(seed=0, shape=SHAPE):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


def pair(seed, shape, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    c = torch.randn(shape, generator=g)
    u = 0.6 * c + 0.5 * torch.randn(shape, generator=g)
    return c.to(dtype), u.to(dtype)


# ---- algebra ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("levels,hw", [(2, (12, 16)), (3, (24, 12)), (4, (64, 64)), (5, (48, 80))])
def test_correction_form_equals_per_level_form(levels, hw):
    """In float64 the correction form on the pyramid of d equals diffusers' per-level form to 1e-12; the fp32 device
    arithmetic is within 1e-5 of it (relative to the largest |g|)."""
    c, u = pair(levels, (3, 2) + hw)
    scales = torch.tensor([[9.0, 4.0, 2.5, 1.5, 1.0][:levels], [3.0, 6.0, 1.0, 2.0, 4.0][:levels], [1.0] * levels])
    want = fdg_fp64(c, u, scales, levels)
    # the correction form in float64
    d = (c.double() - u.double()).numpy()
    w = scales.double().numpy()
    bs = (3, 1, 1, 1)
    G = [d]
    for _ in range(levels - 1):
        G.append(down2(G[-1], np.float64))
    g = u.double().numpy() + w[:, 0].reshape(bs) * d
    if levels > 1:
        E = (w[:, levels - 1] - w[:, levels - 2]).reshape(bs) * G[-1]
        for l in range(levels - 2, 0, -1):
            E = (w[:, l] - w[:, l - 1]).reshape(bs) * G[l] + up2(E, np.float64)
        g = g + up2(E, np.float64)
    scale = np.abs(want).max()
    assert np.abs(g - want).max() <= 1e-12 * scale
    got = fdg_exact(c, u, scales, levels).double().numpy()
    assert np.abs(got - want).max() <= 1e-5 * scale


def test_filters_against_conv_and_interpolate():
    """Down is the 5x5 binomial blur (reflect) followed by half-pixel bilinear 1/2; Up is bilinear x2 followed by the
    blur away from the borders (float64)."""
    import torch.nn.functional as F
    a = torch.randn(1, 1, 16, 20, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
    k1 = torch.tensor([1., 4., 6., 4., 1.], dtype=torch.float64) / 16
    k = (k1[:, None] * k1[None, :])[None, None]
    blur = lambda x: F.conv2d(F.pad(x, (2, 2, 2, 2), mode="reflect"), k)
    down = F.interpolate(blur(a), scale_factor=0.5, mode="bilinear", align_corners=False)
    assert np.abs(down2(a.numpy(), np.float64) - down.numpy()).max() <= 1e-14
    up = blur(F.interpolate(a, scale_factor=2, mode="bilinear", align_corners=False)).numpy()
    assert np.abs(up2(a.numpy(), np.float64)[..., 3:-3, 3:-3] - up[..., 3:-3, 3:-3]).max() <= 1e-14


# ---- the identities --------------------------------------------------------------------------------------------------

def test_one_level_is_the_cfg_combine():
    c, u = pair(1, (2, 3, 7, 5))
    for w in (4.5, 1.0, -2.0):
        assert torch.equal(fdg_exact(c, u, [w], 1), u + w * (c - u))


@pytest.mark.parametrize("levels", [2, 3])
def test_equal_scales_are_one_level(levels):
    c, u = pair(2, (2, 3, 12, 16))
    a = fdg_exact(c, u, [3.25] * levels, levels)
    b = fdg_exact(c, u, [3.25], 1)
    assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_condition_blind_gives_u(dtype):
    _, u = pair(3, (2, 3, 12, 16), dtype)
    assert torch.equal(fdg_exact(u, u.clone(), SCALES, 3), u)


def test_checkerboard_has_no_coarse_levels():
    _, u = pair(4, (1, 2, 12, 16))
    ii, jj = torch.meshgrid(torch.arange(12), torch.arange(16), indexing="ij")
    d = torch.where((ii + jj) % 2 == 0, 1.0, -1.0)
    assert not down2(d.numpy()).any()
    c = u + d
    w0 = SCALES[0]
    assert torch.equal(fdg_exact(c, u, SCALES, 3), u + w0 * ((u + d) - u))


def test_constant_difference_gets_the_coarsest_scale():
    _, u = pair(5, (1, 2, 12, 16))
    c = u + 0.75
    got = fdg_exact(c, u, SCALES, 3)
    want = u.double() + SCALES[-1] * 0.75
    assert float((got.double() - want).abs().max()) <= 1e-5


# ---- sample() against the reference ----------------------------------------------------------------------------------

METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2),
           ("singlestep", 3), ("singlestep_fixed", 2), ("adaptive", 2)]
PER_SAMPLE = torch.tensor([[7.0, 3.5, 1.5], [2.0, 4.0, 1.0]])


@needs_ref
@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("method,order", METHODS)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("cfg", ["shared", "shared-thr", "per_sample"])
def test_sample_matches_reference(fdg_backend, mt, method, order, algo, cfg, capsys):
    import dpm_solver_b200 as new
    thr = cfg.endswith("thr")
    if thr and algo == "dpmsolver":
        pytest.skip("thresholding acts on the data prediction")
    scales = PER_SAMPLE if cfg == "per_sample" else SCALES
    ns = product_schedule(mt)
    calls, ref_calls = [], []
    fn = wrap(mt, ns, scales, model=counted(calls))
    skw = dict(steps=5, order=order, method=method)
    if method == "adaptive":
        skw = dict(order=order, method=method, atol=0.05, rtol=0.1)
    y = new.DPM_Solver(fn, ns, algorithm_type=algo,
                       correcting_x0_fn="dynamic_thresholding" if thr else None).sample(x_T(), **skw)
    yr = reference(mt, algo, scales, thr, ref_calls).sample(x_T(), **skw)
    capsys.readouterr()
    assert len(calls) == len(ref_calls) and all(c == (2 * B,) + SHAPE[1:] for c in calls)
    if method == "adaptive":
        # the host controller's step-size scalars are the reference's to within an fp32 rounding, as for plain CFG
        err = float((y.double() - yr.double()).abs().max() / yr.double().abs().max())
        assert err <= 1e-5, err
        return
    assert torch.equal(y, yr), float((y - yr).abs().max())


@needs_ref
@pytest.mark.parametrize("mt", ["noise", "v", "flow", "edm"])
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
def test_denoise_to_zero_and_inverse(fdg_backend, mt, algo):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    skw = dict(steps=5, order=2, method="multistep", denoise_to_zero=True)
    y = new.DPM_Solver(wrap(mt, ns), ns, algorithm_type=algo).sample(x_T(), **skw)
    yr = reference(mt, algo, SCALES).sample(x_T(), **skw)
    assert torch.equal(y, yr)
    ikw = dict(steps=4, order=2, method="multistep")
    yi = new.DPM_Solver(wrap(mt, ns), ns, algorithm_type=algo).inverse(x_T(1), **ikw)
    yg = new.DPM_Solver(guided_wrap(mt, ns), ns, algorithm_type=algo).inverse(x_T(1), **ikw)
    assert torch.equal(yi, yg)


@pytest.mark.parametrize("kind", ["linear", "cosine"])
def test_continuous_vp_schedules(fdg_backend, kind):
    import dpm_solver_b200 as new
    ns = product_schedule("noise", kind)
    y = new.DPM_Solver(wrap("noise", ns), ns).sample(x_T(), steps=5, order=2)
    yg = new.DPM_Solver(guided_wrap("noise", ns), ns).sample(x_T(), steps=5, order=2)
    assert torch.equal(y, yg)


def test_return_intermediate_and_hooks(fdg_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    fx0 = lambda x0, t: 0.9 * x0
    fxt = lambda x, t, step: x * 0.999
    kw = dict(steps=4, order=2, method="multistep", return_intermediate=True)
    y, inter = new.DPM_Solver(wrap("v", ns), ns, correcting_x0_fn=fx0, correcting_xt_fn=fxt).sample(x_T(), **kw)
    yg, interg = new.DPM_Solver(guided_wrap("v", ns), ns, correcting_x0_fn=fx0, correcting_xt_fn=fxt).sample(
        x_T(), **kw)
    assert torch.equal(y, yg) and len(inter) == len(interg)
    assert all(torch.equal(a, b) for a, b in zip(inter, interg))


# ---- other solver paths ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("thr", [False, True])
def test_unipc_matches_the_guided_network(fdg_backend, mt, algo, thr):
    import dpm_solver_b200 as new
    if thr and algo == "dpmsolver":
        pytest.skip("thresholding acts on the data prediction")
    ns = product_schedule(mt)
    kw = dict(algorithm_type=algo, variant="bh2", correcting_x0_fn="dynamic_thresholding" if thr else None)
    y = new.UniPC(wrap(mt, ns, PER_SAMPLE), ns, **kw).sample(x_T(), steps=5, order=3)
    yg = new.UniPC(guided_wrap(mt, ns, PER_SAMPLE), ns, **kw).sample(x_T(), steps=5, order=3)
    assert torch.equal(y, yg)


def test_per_sample_rows_equal_their_shared_runs(fdg_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    x = x_T(2)
    y = new.DPM_Solver(wrap("noise", ns, PER_SAMPLE), ns).sample(x, steps=5, order=2)
    for b in range(B):
        yb = new.DPM_Solver(wrap("noise", ns, PER_SAMPLE[b].tolist(), b=1), ns).sample(x[b:b + 1], steps=5, order=2)
        assert torch.equal(y[b:b + 1], yb)


def test_one_level_fp32_noise_run_equals_plain_cfg(fdg_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    for algo in ("dpmsolver", "dpmsolver++"):
        y = new.DPM_Solver(wrap("noise", ns, [4.5]), ns, algorithm_type=algo).sample(x_T(), steps=5, order=2)
        fn = new.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B, 1),
                               unconditional_condition=torch.zeros(B, 1), guidance_scale=4.5)
        assert torch.equal(y, new.DPM_Solver(fn, ns, algorithm_type=algo).sample(x_T(), steps=5, order=2))


@pytest.mark.parametrize("state_dtype", [None, torch.bfloat16, torch.float16])
def test_condition_blind_run_equals_unguided(fdg_backend, state_dtype):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    y = new.DPM_Solver(wrap("noise", ns, model=blind), ns, state_dtype=state_dtype).sample(x_T(), steps=5, order=2)
    fn = new.model_wrapper(lambda x, t: blind(x, t, None), ns)
    assert torch.equal(y, new.DPM_Solver(fn, ns, state_dtype=state_dtype).sample(x_T(), steps=5, order=2))


@pytest.mark.parametrize("shape,scales", [((2, 4, 2, 12, 12), SCALES), ((2, 1, 96, 64), [5.0, 4.0, 3.0, 2.0, 1.0]),
                                          ((2, 2, 24, 40), [6.0, 2.0, 1.0, 0.5]), ((2, 3, 7, 9), [3.0])])
def test_shapes(fdg_backend, shape, scales):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    x = x_T(3, shape)
    y = new.DPM_Solver(wrap("noise", ns, scales), ns).sample(x, steps=3, order=2)
    yg = new.DPM_Solver(guided_wrap("noise", ns, scales), ns).sample(x, steps=3, order=2)
    assert torch.equal(y, yg)


# ---- calls and counts ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_direct_model_fn_call(fdg_backend, mt):
    ns = product_schedule(mt)
    x, t = x_T(3), torch.full((B,), 0.5)
    assert torch.equal(wrap(mt, ns, PER_SAMPLE)(x, t), guided_wrap(mt, ns, PER_SAMPLE)(x, t))
    t2 = torch.tensor([0.5, 0.3])
    assert torch.equal(wrap(mt, ns)(x, t2), guided_wrap(mt, ns)(x, t2))


def test_launch_and_network_call_counts(fdg_backend):
    """Per evaluation: one network call on 2B rows and one pyramid launch more than the run on the guided network; plus
    one launch that doubles the first input (every later doubled input is written by the step that makes it)."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    for thr in (False, True):
        calls, gcalls = [], []
        kw = dict(correcting_x0_fn="dynamic_thresholding" if thr else None)
        s = new.DPM_Solver(wrap("noise", ns, model=counted(calls)), ns, **kw)
        g = guided_net(net, torch.zeros(B, 1), torch.ones(B, 1), SCALES, gcalls)
        s0 = new.DPM_Solver(new.model_wrapper(lambda x, t: g(x, t), ns), ns, **kw)
        n0 = fdg_backend.launch_count()
        s0.sample(x_T(), steps=5, order=2)
        base = fdg_backend.launch_count() - n0
        n1 = fdg_backend.launch_count()
        s.sample(x_T(), steps=5, order=2)
        assert fdg_backend.launch_count() - n1 == base + len(calls) + 1
        assert len(calls) == len(gcalls) == 5 and all(c == (2 * B,) + SHAPE[1:] for c in calls)


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    from dpm_solver_b200 import ops
    from dpm_solver_b200.distributed import shard_batch
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ops.set_backend(FDGOracle())
        import dpm_solver_b200 as new
        ns = product_schedule("noise")
        scales = torch.tensor([[7.0, 3.5, 1.5], [2.0, 4.0, 1.0], [1.0, 1.0, 5.0], [3.0, 3.0, 3.0]])
        x = shard_batch(x_T(4, (4,) + SHAPE[1:]), rank, world)
        fn = wrap("noise", ns, shard_batch(scales, rank, world), b=x.shape[0])
        y = new.DPM_Solver(fn, ns, plan_broadcast=True).sample(x, steps=4, order=2)
        q.put((rank, y))
    finally:
        dist.destroy_process_group()


def test_batch_sharding_needs_no_collective(fdg_backend):
    """Two gloo ranks of two samples each, the [B, N] scales split like the batch, equal the unsharded run of four."""
    import socket
    import torch.multiprocessing as mp
    import dpm_solver_b200 as new
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    ns = product_schedule("noise")
    scales = torch.tensor([[7.0, 3.5, 1.5], [2.0, 4.0, 1.0], [1.0, 1.0, 5.0], [3.0, 3.0, 3.0]])
    y = new.DPM_Solver(wrap("noise", ns, scales, b=4), ns).sample(x_T(4, (4,) + SHAPE[1:]), steps=4, order=2)
    assert torch.equal(torch.cat([got[0], got[1]]), y)


# ---- rejections ------------------------------------------------------------------------------------------------------

def _rejections(calls):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    m = counted(calls)
    cf = dict(guidance_type="classifier-free", condition=torch.ones(B, 1), unconditional_condition=torch.zeros(B, 1))
    mw = lambda **kw: new.model_wrapper(m, ns, **{**cf, **kw})
    yield lambda: new.model_wrapper(m, ns, guidance_type="uncond", fdg_scales=SCALES)
    yield lambda: new.model_wrapper(m, ns, guidance_type="classifier-free", condition=torch.ones(B, 1),
                                    fdg_scales=SCALES)
    yield lambda: mw(condition=[torch.ones(B, 1), torch.ones(B, 1)], guidance_scale=[2.0, 3.0], fdg_scales=SCALES)
    yield lambda: mw(guidance_mask=[torch.ones(B, 1, 1, 1)], condition=[torch.ones(B, 1)], guidance_scale=[2.0],
                     fdg_scales=SCALES)
    yield lambda: mw(guidance_rescale=0.7, fdg_scales=SCALES)
    yield lambda: mw(apg_eta=0.0, fdg_scales=SCALES)
    yield lambda: mw(cfg_zero_star=True, fdg_scales=SCALES)
    yield lambda: mw(cfg_pp=True, fdg_scales=SCALES)
    yield lambda: mw(tcfg=True, fdg_scales=SCALES)
    yield lambda: mw(guidance_scale=7.5, fdg_scales=SCALES)
    yield lambda: mw(guidance_scale=torch.tensor([2.0, 3.0]), fdg_scales=SCALES)
    yield lambda: mw(fdg_scales=[])
    yield lambda: mw(fdg_scales=[1.0] * 6)
    yield lambda: mw(fdg_scales=torch.ones(B, 2, 3))
    yield lambda: new.DPM_Solver(mw(fdg_scales=torch.ones(3, 3)), ns).sample(x_T(), steps=3)      # 3 rows for B = 2
    yield lambda: new.DPM_Solver(mw(fdg_scales=SCALES), ns).sample(x_T(0, (2, 3, 10, 16)), steps=3)   # 10/4 < 3
    yield lambda: new.DPM_Solver(mw(fdg_scales=[1.0] * 4), ns).sample(x_T(0, (2, 3, 16, 16)), steps=3)  # 16/8 < 3
    yield lambda: new.DPM_Solver(mw(fdg_scales=[1.0]), ns).sample(x_T(0, (2, 3, 130, 130)), steps=3)  # H*W > 16384
    yield lambda: new.DPM_Solver(mw(fdg_scales=[1.0]), ns).sample(x_T(0, (2, 48)), steps=3)          # x.dim() < 4
    yield lambda: new.UniPC(mw(fdg_scales=SCALES), ns).sample(x_T(0, (2, 3, 10, 16)), steps=3)
    yield lambda: new.DPM_Solver(mw(fdg_scales=SCALES), ns, algorithm_type="dpmsolver", reference_rounding=True)
    yield lambda: mw(fdg_scales=SCALES)(x_T(0, (2, 3, 10, 16)), torch.full((B,), 0.5))


def test_rejections_launch_nothing(fdg_backend):
    n, calls = 0, []
    for call in _rejections(calls):
        before = fdg_backend.launch_count()
        with pytest.raises(ValueError):
            call()
        assert fdg_backend.launch_count() == before and calls == [], n
        n += 1
    assert n == 22


def test_size_rule_lives_in_the_library():
    from dpm_solver_b200 import _lib, ops
    lib = _lib.lib()
    assert lib.dpm_fdg_supported(128, 128, 5, 1) == 0 and lib.dpm_fdg_supported(64, 64, 5, 1) == 0
    assert lib.dpm_fdg_supported(256, 256, 1, 1) != 0 and lib.dpm_fdg_supported(24, 24, 5, 1) != 0
    assert lib.dpm_fdg_supported(2 ** 32, 2 ** 32, 1, 0) != 0       # (a product that would wrap to 0)
    ops.fdg_check((1, 4, 24, 24), 4)
    with pytest.raises(ValueError, match="divisible"):
        ops.fdg_check((1, 4, 24, 24), 5)


def test_tensor_scales_are_converted_per_version(fdg_backend):
    """A 1-D tensor and a list of one-element tensors are read as tensors: an in-place write to the 1-D tensor or to
    any one of the listed tensors takes effect at the next run, and both give the run of the same numbers."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    want = new.DPM_Solver(wrap("noise", ns, SCALES), ns).sample(x_T(), steps=3, order=2)
    t = torch.tensor(SCALES)
    s = new.DPM_Solver(wrap("noise", ns, t), ns)
    assert torch.equal(s.sample(x_T(), steps=3, order=2), want)
    ts = [torch.tensor(v) for v in SCALES[:2]] + [torch.tensor([SCALES[2]], dtype=torch.float64)]
    listed = new.DPM_Solver(wrap("noise", ns, ts), ns)
    assert torch.equal(listed.sample(x_T(), steps=3, order=2), want)
    t.copy_(torch.tensor([2.0, 1.0, 0.5]))
    want2 = new.DPM_Solver(wrap("noise", ns, [2.0, 1.0, 0.5]), ns).sample(x_T(), steps=3, order=2)
    assert torch.equal(s.sample(x_T(), steps=3, order=2), want2)
    for k, v in ((0, 2.0), (1, 1.0), (2, 0.5)):          # one listed tensor at a time, each write seen at once
        ts[k].fill_(v)
        scales = [float(u) for u in ts]
        want_k = new.DPM_Solver(wrap("noise", ns, scales), ns).sample(x_T(), steps=3, order=2)
        assert torch.equal(listed.sample(x_T(), steps=3, order=2), want_k), k
    assert torch.equal(listed.sample(x_T(), steps=3, order=2), want2)
