"""Frequency-decoupled guidance on the H100: dpm_fdg_guided bit for bit against tests/fdg_oracle.fdg_exact over dtypes,
levels, plane shapes, plane counts, layouts, per-sample scales and IEEE edges, beyond 2^31 elements; sample() on the
device against the numpy executor; a condition-blind run against the unmodified reference's unguided run."""
import pytest
import torch

from fdg_oracle import FDGOracle, fdg_exact
from oracle import ref_loader

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


@pytest.fixture(scope="module")
def cuda_be():
    from dpm_solver_b200 import ops
    return ops.CudaBackend()


def pair(seed, shape, dtype):
    g = torch.Generator().manual_seed(seed)
    c = torch.randn(shape, generator=g) * 2.0
    u = 0.6 * c + torch.randn(shape, generator=g)
    return c.to(dtype), u.to(dtype)


def scale_rows(levels, B, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(B, levels, generator=g) * 12.0 - 2.0).float()


def same_bits(a, b):
    """Equal values bit for bit, any NaN matching any NaN (a NaN's payload is not part of the contract)."""
    a, b = a.cpu().float(), b.cpu().float()
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    return torch.equal(a[~na].view(torch.int32), b[~nb].view(torch.int32))


def run(be, c, u, scales, levels):
    sc = scales.to(DEV) if torch.is_tensor(scales) else scales
    return be.fdg_guided(c.to(DEV) if not c.is_cuda else c, u.to(DEV) if not u.is_cuda else u, sc, levels)


PLANES = [((64, 64), 5), ((128, 128), 5), ((96, 64), 5), ((24, 24), 4), ((12, 20), 3)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("hw,max_levels", PLANES)
@pytest.mark.parametrize("per_sample", [False, True])
def test_pass_bit_exact(cuda_be, dtype, hw, max_levels, per_sample):
    for levels in range(1, max_levels + 1):
        for B, C in ((1, 1), (3, 4), (2, 16)):
            c, u = pair(levels * 7 + B, (B, C) + hw, dtype)
            scales = scale_rows(levels, B, levels) if per_sample else [10.0, 5.0, 2.5, 1.0, 3.0][:levels]
            got = run(cuda_be, c, u, scales, levels)
            assert got.dtype == dtype and got.shape == c.shape
            assert same_bits(got, fdg_exact(c, u, scales, levels)), (levels, B, C)


@pytest.mark.parametrize("dtype", DTYPES)
def test_thousands_of_planes(cuda_be, dtype):
    c, u = pair(11, (640, 4, 64, 64), dtype)            # 2560 planes
    scales = scale_rows(4, 640, 3)
    assert same_bits(run(cuda_be, c, u, scales, 4), fdg_exact(c, u, scales, 4))
    c, u = pair(12, (16, 16, 128, 128), dtype)          # 256 planes of the largest size
    assert same_bits(run(cuda_be, c, u, [10.0, 5.0], 2), fdg_exact(c, u, [10.0, 5.0], 2))


@pytest.mark.parametrize("dtype", DTYPES)
def test_layouts(cuda_be, dtype):
    c, u = pair(13, (3, 4, 64, 96), dtype)
    want = fdg_exact(c, u, [8.0, 4.0, 2.0], 3)
    cl = run(cuda_be, c.to(DEV).contiguous(memory_format=torch.channels_last),
             u.to(DEV).contiguous(memory_format=torch.channels_last), [8.0, 4.0, 2.0], 3)
    assert cl.is_contiguous(memory_format=torch.channels_last) and same_bits(cl, want)
    n = c.numel()
    cb, ub = torch.empty(n + 1, dtype=dtype, device=DEV), torch.empty(n + 1, dtype=dtype, device=DEV)
    cb[1:] = c.to(DEV).reshape(-1)
    ub[1:] = u.to(DEV).reshape(-1)
    off = run(cuda_be, cb[1:].view(c.shape), ub[1:].view(c.shape), [8.0, 4.0, 2.0], 3)
    assert same_bits(off, want)
    # 5-D, channels_last_3d (planes not indexed by one stride: a copy) and a transposed view (the strided path)
    c5, u5 = pair(14, (2, 3, 2, 24, 24), dtype)
    want5 = fdg_exact(c5, u5, [6.0, 3.0, 1.0, 2.0], 4)
    assert same_bits(run(cuda_be, c5, u5, [6.0, 3.0, 1.0, 2.0], 4), want5)
    cl3 = lambda t: t.to(DEV).contiguous(memory_format=torch.channels_last_3d)
    assert same_bits(run(cuda_be, cl3(c5), cl3(u5), [6.0, 3.0, 1.0, 2.0], 4), want5)
    ct, ut = c.transpose(-1, -2).contiguous().to(DEV).transpose(-1, -2), u.transpose(-1, -2).contiguous().to(DEV)
    assert same_bits(run(cuda_be, ct, ut.transpose(-1, -2), [8.0, 4.0, 2.0], 3), want)


@pytest.mark.parametrize("dtype", DTYPES)
def test_ieee_edges(cuda_be, dtype):
    c, u = pair(15, (4, 4, 24, 24), dtype)
    specials = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -1e-42, 3e-39])
    g = torch.Generator().manual_seed(16)
    for t in (c, u):
        idx = torch.randint(0, t.numel(), (60,), generator=g)
        t.view(-1)[idx] = specials[torch.randint(0, len(specials), (60,), generator=g)].to(dtype)
    c[0] = 0.0
    u[0] = -0.0
    for scales in ([0.0, -0.0, 1.0], [float("inf"), 1.0, 2.0], [1e-40, float("nan"), 3.0]):
        assert same_bits(run(cuda_be, c, u, scales, 3), fdg_exact(c, u, scales, 3))
    rows = scale_rows(3, 4, 4)
    rows[1, 1] = float("nan")
    rows[2, 0] = float("-inf")
    rows[3] = torch.tensor([1e-41, -0.0, 2e-39])
    assert same_bits(run(cuda_be, c, u, rows, 3), fdg_exact(c, u, rows, 3))


def test_deterministic_and_batch_position_independent(cuda_be):
    c, u = pair(17, (8, 4, 64, 64), torch.bfloat16)
    c, u = c.to(DEV), u.to(DEV)
    rows = scale_rows(3, 8, 5).to(DEV)
    a = cuda_be.fdg_guided(c, u, rows, 3)
    b = cuda_be.fdg_guided(c, u, rows, 3)
    assert torch.equal(a, b)
    perm = torch.tensor([5, 2, 7, 0, 1, 6, 3, 4], device=DEV)
    p = cuda_be.fdg_guided(c[perm].contiguous(), u[perm].contiguous(), rows[perm].contiguous(), 3)
    assert torch.equal(p, a[perm])


def test_beyond_two_to_the_31_elements(cuda_be):
    """One launch over 2^31 + 16384 bf16 elements (131073 planes of 128 x 128): sampled planes equal fdg_exact."""
    planes = 131073
    shape = (planes, 1, 128, 128)
    gen = torch.Generator(device=DEV).manual_seed(18)
    c = torch.randn(shape, device=DEV, dtype=torch.bfloat16, generator=gen)
    u = torch.randn(shape, device=DEV, dtype=torch.bfloat16, generator=gen)
    rows = (torch.rand(planes, 3, device=DEV, generator=gen) * 8.0).contiguous()
    g = cuda_be.fdg_guided(c, u, rows, 3)
    torch.cuda.synchronize()
    for p in (0, 1, 65535, 65536, 131071, planes - 1):
        sl = slice(p, p + 1)
        assert same_bits(g[sl], fdg_exact(c[sl].cpu(), u[sl].cpu(), rows[sl].cpu(), 3)), p
    del c, u, g


# ---- sample() on the device against the executor ---------------------------------------------------------------------

# (rounded elementwise ops only, so that the network gives the same bits on the device and on the CPU)
def net(x, t, c):
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.4 * x + cc * (0.1 * (x * x) - 0.2 * x) - 0.1


def blind(x, t, c):
    return 0.4 * x + 0.05 * (x * x) - 0.1


def schedule(mt):
    import dpm_solver_b200 as new
    from cases import make_betas
    if mt == "flow":
        return new.NoiseScheduleFlow(shift=3.0)
    if mt == "edm":
        return new.NoiseScheduleEDM()
    return new.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def solve(device, mt="noise", scales=(7.0, 3.5, 1.5), shape=(2, 4, 32, 32), solver="dpm", model=net, state_dtype=None,
          thr=False, skw=None, seed=0, calls=2):
    import dpm_solver_b200 as new
    ns = schedule(mt)
    B = shape[0]
    sc = scales.to(device) if torch.is_tensor(scales) else list(scales)
    fn = new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free",
                           condition=torch.ones(B, 1, device=device), unconditional_condition=torch.zeros(B, 1,
                                                                                                       device=device),
                           fdg_scales=sc)
    kw = dict(correcting_x0_fn="dynamic_thresholding" if thr else None)
    s = (new.UniPC(fn, ns, state_dtype=state_dtype, **kw) if solver == "unipc"
         else new.DPM_Solver(fn, ns, state_dtype=state_dtype, **kw))
    x = torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(device)
    out = [s.sample(x, **(skw or dict(steps=5, order=2))) for _ in range(calls)]
    return out


def on(backend, fn):
    from dpm_solver_b200 import ops
    old = ops._backend
    ops.set_backend(backend)
    try:
        return fn()
    finally:
        ops.set_backend(old)


CASES = [dict(), dict(scales=torch.tensor([[7.0, 3.5, 1.5], [2.0, 4.0, 1.0]])), dict(mt="flow"), dict(mt="edm"), dict(thr=True), dict(solver="unipc", skw=dict(steps=5, order=3)),
         dict(skw=dict(steps=5, order=3, method="singlestep", return_intermediate=True)),
         dict(mt="v", skw=dict(steps=5, order=2, denoise_to_zero=True))]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_sample_matches_executor(cuda_be, case):
    kw = CASES[case]
    got = on(cuda_be, lambda: solve(DEV, **kw))
    want = on(FDGOracle(), lambda: solve("cpu", **kw))
    for a, b in zip(got, want):
        if isinstance(a, tuple):
            assert torch.equal(a[0].cpu(), b[0]) and all(torch.equal(p.cpu(), q) for p, q in zip(a[1], b[1]))
        else:
            assert torch.equal(a.cpu(), b), float((a.cpu() - b).abs().max())


def test_bf16_state(cuda_be):
    """bf16 state: the network itself then computes in bf16, where torch's CPU and CUDA kernels round a python scalar
    differently; a fresh solver repeats the device run bit for bit and the executor's run is within bf16 rounding."""
    a = on(cuda_be, lambda: solve(DEV, state_dtype=torch.bfloat16))
    b = on(cuda_be, lambda: solve(DEV, state_dtype=torch.bfloat16, calls=1))
    assert torch.equal(a[0], a[1]) and torch.equal(a[0], b[0])
    w = on(FDGOracle(), lambda: solve("cpu", state_dtype=torch.bfloat16, calls=1))[0].float()
    assert float((a[0].float().cpu() - w).abs().max() / w.abs().max()) <= 2e-2


def bounded(x, t, c):
    """A network whose guidance term stays bounded, so that the adaptive solver takes few steps."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.4 * x + cc * (0.3 * x / (1.0 + x * x)) - 0.1


def test_device_adaptive_controller(cuda_be):
    """The device controller's run equals the one on a network that returns the FDG output g, on the same
    controller."""
    import dpm_solver_b200 as new
    from fdg_oracle import guided_net
    ns = schedule("noise")
    x = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(4)).to(DEV)
    kw = dict(order=2, method="adaptive", atol=0.05, rtol=0.1)
    fn = new.model_wrapper(bounded, ns, guidance_type="classifier-free", condition=torch.ones(2, 1, device=DEV),
                           unconditional_condition=torch.zeros(2, 1, device=DEV), fdg_scales=[3.0, 2.0, 1.5])
    y = on(cuda_be, lambda: new.DPM_Solver(fn, ns).sample(x.clone(), **kw))
    g = guided_net(bounded, torch.zeros(2, 1), torch.ones(2, 1), [3.0, 2.0, 1.5])
    gnet = lambda xx, tt: g(xx.cpu(), tt.cpu()).to(xx.device)
    yg = on(cuda_be, lambda: new.DPM_Solver(new.model_wrapper(gnet, ns), ns).sample(x.clone(), **kw))
    assert torch.equal(y, yg)


def test_capture_replay_follows_rewritten_scales(cuda_be):
    import dpm_solver_b200 as new
    ns = schedule("noise")
    B, shape = 2, (2, 4, 64, 64)
    rows = torch.tensor([[7.0, 3.5, 1.5], [2.0, 4.0, 1.0]], device=DEV)
    fn = new.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B, 1, device=DEV),
                           unconditional_condition=torch.zeros(B, 1, device=DEV), fdg_scales=rows)
    s = new.DPM_Solver(fn, ns)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1)).to(DEV)
    replay = on(cuda_be, lambda: s.capture(x, steps=5, order=2))
    y1 = on(cuda_be, lambda: replay(x)).clone()
    rows.copy_(torch.tensor([[1.0, 5.0, 9.0], [3.0, 3.0, 0.5]], device=DEV))
    y2 = on(cuda_be, lambda: replay(x)).clone()
    torch.cuda.synchronize()
    for y, sc in ((y1, [[7.0, 3.5, 1.5], [2.0, 4.0, 1.0]]), (y2, [[1.0, 5.0, 9.0], [3.0, 3.0, 0.5]])):
        want = on(FDGOracle(), lambda: solve("cpu", scales=torch.tensor(sc), shape=shape, seed=1, calls=1))[0]
        assert torch.equal(y.cpu(), want)


@pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")
def test_condition_blind_run_equals_reference_unguided(cuda_be):
    """fp32 [4, 4, 64, 64]: FDG on a network blind to the condition equals the unmodified reference's unguided run."""
    ref = ref_loader.load("dpm_solver_pytorch")
    from cases import make_betas
    shape = (4, 4, 64, 64)
    y = on(cuda_be, lambda: solve(DEV, model=blind, shape=shape, scales=(10.0, 5.0, 2.0, 1.0), calls=1))[0]
    rns = ref.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    x = torch.randn(shape, generator=torch.Generator().manual_seed(0))
    yr = ref.DPM_Solver(ref.model_wrapper(lambda xx, tt: blind(xx, tt, None), rns), rns).sample(x, steps=5, order=2)
    assert torch.equal(y.cpu(), yr), float((y.cpu() - yr).abs().max())
