"""The in-kernel Gaussian noise (csrc/philox.cu) against torch.randn drawn on the same GPU from the same state.

`DPM_Solver.add_noise(x, t)` without `noise=` and the DiffEdit corrector draw their normals inside `k_noise_philox`,
which replays ATen's launch geometry for an fp32 randn of the same size. So for the generator's (seed, offset) the
values must equal torch.randn's bit for bit, and the generator must end where randn leaves it. The sizes sit on
every edge of that geometry, derived from the device rather than fixed for one SKU:
- the 256-thread block, and the grid saturating at #SM * maxThreadsPerSM/256 blocks, i.e. G threads;
- the counter offset, which steps every 4G elements;
- ATen's split of a tensor beyond 2^29 fp32 elements (no 32-bit byte offsets) into halves, each drawn as its own
  launch with its own grid and philox state.
Every case keeps its peak device memory at or below 12 GiB."""
import ctypes as C

import pytest
import torch

from cases import make_betas

pytestmark = pytest.mark.gpu

PEAK_BYTES = 12 << 30
SPLIT = 1 << 29          # the largest fp32 tensor ATen draws in one launch: 1 + (2^29 - 1) * 4 <= INT32_MAX
DPM_F32, DPM_ERR_ARG = 0, -1
_BITS = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}


def _threads(dev):
    """G: the threads of ATen's saturated randn grid on `dev`."""
    p = torch.cuda.get_device_properties(dev)
    return p.multi_processor_count * (p.max_threads_per_multi_processor // 256) * 256


@pytest.fixture()
def dev(cuda_backend):
    d = torch.device("cuda", torch.cuda.current_device())
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(d)
    yield d
    peak = torch.cuda.max_memory_allocated(d)
    torch.cuda.empty_cache()
    assert peak <= PEAK_BYTES, f"peak device memory {peak / 2**30:.2f} GiB"


def _sched(mod):
    return mod.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def _data(shape, seed, dev, dtype=torch.float32):
    """Seeded test data drawn on the device from a private generator (the default one is left alone)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, device=dev, generator=g).to(dtype)


def _bits_mismatch(got, want, chunk=1 << 26):
    """None if two tensors of one dtype hold the same bits (NaN: same positions, any payload), else a description."""
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    a, b = got.reshape(-1), want.reshape(-1)
    for i in range(0, a.numel(), chunk):
        ca, cb = a[i:i + chunk], b[i:i + chunk]
        nan_a, nan_b = torch.isnan(ca), torch.isnan(cb)
        ia = torch.where(nan_a, 0, ca.view(_BITS[ca.dtype]))
        ib = torch.where(nan_b, 0, cb.view(_BITS[cb.dtype]))
        bad = (ia != ib) | (nan_a != nan_b)
        if bool(bad.any()):
            j = int(bad.nonzero()[0])
            return (f"{int(bad.sum())}+ of {a.numel()} elements differ, first at {i + j}: "
                    f"{float(ca[j])} vs {float(cb[j])}")
    return None


def _assert_same(got, want):
    msg = _bits_mismatch(got, want)
    assert msg is None, msg


def _offset_after_randn(gen, start, shape, dev):
    """Restore `start`, draw torch.randn(shape) -> (noise, offset after it, the next torch.randn(7))."""
    gen.set_state(start)
    noise = torch.randn(shape, device=dev, generator=gen)
    off = gen.get_offset()
    nxt = torch.randn(7, device=dev, generator=gen)
    return noise, off, nxt


# ---- (a) raw noise: alpha = 0, sigma = 1 leaves the noise itself ---------------------------------------------------
def _raw_noise_check(be, T, n, dev, seed, out_dtype=torch.float32, pre=5):
    """add_noise_philox on zeros with alpha = 0, sigma = 1 vs torch.randn((T, n)) from the same generator state.
    Returns the list of what differs (values, the offset after the draw, the next draw)."""
    gen = torch.cuda.default_generators[dev.index]
    with torch.cuda.device(dev):
        torch.cuda.manual_seed(seed)
        torch.randn(pre, device=dev)                                   # start at a non-zero philox offset
    start = gen.get_state()
    assert gen.get_offset() > 0
    x = torch.zeros(n, dtype=out_dtype, device=dev)
    got = be.add_noise_philox(x, [0.0] * T, [1.0] * T, out_dtype)
    del x
    off = gen.get_offset()
    nxt = torch.randn(7, device=dev, generator=gen)
    want, want_off, want_nxt = _offset_after_randn(gen, start, (T, n), dev)
    bad = []
    if off != want_off:
        bad.append(f"generator offset {off}, torch.randn leaves {want_off}")
    if not torch.equal(nxt, want_nxt):
        bad.append("the next torch.randn(7) differs")
    chunk = 1 << 26
    g, w = got.reshape(-1), want.reshape(-1)
    for i in range(0, g.numel(), chunk):          # randn(...).to(out_dtype), a chunk at a time
        msg = _bits_mismatch(g[i:i + chunk], w[i:i + chunk].to(out_dtype))
        if msg is not None:
            bad.append(f"values (from element {i}): {msg}")
            break
    return bad


def _factorings(numel):
    """(T, n) pairs with T * n = numel: T = 1 and every T in {2, 3, 5, 16} that divides (at most one above 2^24)."""
    ts = [t for t in (16, 5, 3, 2) if numel % t == 0]
    if numel > 1 << 24:
        ts = ts[:1]
    return [(1, numel)] + [(t, numel // t) for t in ts]


_SIZES = {str(k): (lambda G, k=k: k) for k in list(range(1, 10)) + [255, 256, 257, 1023, 1024, 1025]}
_SIZES.update({f"G{d:+d}": (lambda G, d=d: G + d) for d in (-1, 0, 1, 16)})          # grid saturation; 16 * odd
_SIZES.update({f"{k}*4G{d:+d}": (lambda G, k=k, d=d: 4 * k * G + d) for k in (1, 2, 3) for d in (-1, 0, 1)})
_SIZES.update({f"2^24{d:+d}": (lambda G, d=d: (1 << 24) + d) for d in (-1, 0, 1)})
_SIZES.update({"2^29": lambda G: SPLIT, "2^29+3": lambda G: SPLIT + 3, "2^29+4": lambda G: SPLIT + 4})


@pytest.mark.parametrize("size", list(_SIZES))
def test_raw_noise_is_torch_randn(cuda_backend, dev, size):
    """Bits, the generator offset after the draw and the draw after it, for every (T, n) factoring of the size.
    2^29 elements is one launch; 2^29 + 3 and 2^29 + 4 are split in two (odd and even halves)."""
    G = _threads(dev)
    numel = _SIZES[size](G)
    for T, n in _factorings(numel):
        bad = _raw_noise_check(cuda_backend, T, n, dev, seed=numel % 100003 + T,
                               pre=1 + (numel * 7919 + T) % (8 * G))
        torch.cuda.empty_cache()
        assert not bad, f"T={T}, n={n}: " + "; ".join(bad)


def test_raw_noise_four_pieces(cuda_backend, dev):
    """2^30 + 2^28 + 1 elements: ATen splits twice, four pieces. bf16 output against randn().bfloat16() keeps the
    footprint under the memory bound."""
    numel = (1 << 30) + (1 << 28) + 1
    bad = _raw_noise_check(cuda_backend, 3, numel // 3, dev, seed=31, out_dtype=torch.bfloat16, pre=1000)
    assert not bad, "; ".join(bad)


def test_raw_noise_64bit_seed(cuda_backend, dev):
    """curand_init takes the generator's full 64-bit seed."""
    G = _threads(dev)
    for T, n in ((1, 4 * G + 1), (5, 2 * G + 1)):
        bad = _raw_noise_check(cuda_backend, T, n, dev, seed=(1 << 40) + 12345, pre=77)
        assert not bad, f"T={T}, n={n}: " + "; ".join(bad)


def test_one_launch_up_to_two_pow_29_and_one_per_piece_above(cuda_backend, dev):
    be = cuda_backend
    for numel, launches in ((SPLIT, 1), (SPLIT + 4, 2)):
        x = torch.zeros(numel, dtype=torch.bfloat16, device=dev)
        before = be.launch_count()
        out = be.add_noise_philox(x, [0.0], [1.0], torch.bfloat16)
        assert be.launch_count() - before == launches
        del x, out
        torch.cuda.empty_cache()


# ---- (b) the value chain ---------------------------------------------------------------------------------------
_SPECIALS = [float("inf"), float("-inf"), float("nan"), 0.0, -0.0, 1e-40, -2.5e-39, 1.1754944e-38, 65504.0,
             -65504.0, 7e4, -1e5, 3e38]


def _with_specials(x):
    """x (fp32) with +-inf, NaN, +-0, fp32 subnormals and values at and beyond fp16's range, spread over the tensor."""
    flat = x.reshape(-1)
    for k, v in enumerate(_SPECIALS):
        flat[k * 997 % flat.numel()::4099] = v
    return x


_CHAINS = [(torch.float32, torch.float32), (torch.bfloat16, torch.float32), (torch.bfloat16, torch.bfloat16),
           (torch.float16, torch.float32), (torch.float16, torch.float16)]


@pytest.mark.parametrize("T", [1, 5, 16])
@pytest.mark.parametrize("x_dtype,out_dtype", _CHAINS, ids=lambda d: str(d).replace("torch.", ""))
def test_add_noise_value_chain(cuda_backend, dev, x_dtype, out_dtype, T):
    """DPM_Solver.add_noise(x, t) == the explicit-noise path fed torch.randn from the same state, bit for bit (NaN in
    the same places); and == the unmodified reference's add_noise on CPU, rounded to the output dtype."""
    import dpm_solver_b200 as new
    from oracle import ref_loader
    ns = _sched(new)
    s = new.DPM_Solver(None, ns, state_dtype=None if out_dtype == torch.float32 else out_dtype)
    shape = (5, 4, 64, 65)                     # T = 16: beyond 4G noise elements on an H100
    x = _with_specials(_data(shape, 11 + T, dev) * 3).to(x_dtype)
    t = torch.linspace(1e-3, 1.0, T, device=dev) if T > 1 else torch.tensor([0.37], device=dev)
    gen = torch.cuda.default_generators[dev.index]
    torch.cuda.manual_seed(500 + T)
    torch.randn(3, device=dev)
    start = gen.get_state()
    before = cuda_backend.launch_count()
    got = s.add_noise(x, t)
    assert cuda_backend.launch_count() == before + 1
    off = gen.get_offset()
    noise, want_off, _ = _offset_after_randn(gen, start, (T, *shape), dev)
    assert off == want_off
    want = s.add_noise(x, t, noise=noise)
    assert got.dtype == want.dtype == out_dtype and got.shape == want.shape
    _assert_same(got, want)
    if ref_loader.available():
        ref = ref_loader.load("dpm_solver_pytorch")
        want_cpu = ref.DPM_Solver(None, _sched(ref)).add_noise(x.cpu(), t.cpu(), noise=noise.cpu())
        _assert_same(got.cpu(), want_cpu.to(out_dtype))


# ---- (c) end to end at a split size ----------------------------------------------------------------------------
def test_add_noise_end_to_end_beyond_two_pow_29(cuda_backend, dev):
    """3 labels on a bf16 x of 1.9e8 elements: 5.7e8 noise elements, two pieces."""
    import dpm_solver_b200 as new
    s = new.DPM_Solver(None, _sched(new))
    x = _data((45, 4, 1024, 1024), 3, dev, torch.bfloat16)
    t = torch.tensor([0.9, 0.4, 0.02], device=dev)
    assert 3 * x.numel() > SPLIT
    gen = torch.cuda.default_generators[dev.index]
    torch.cuda.manual_seed(2718)
    torch.randn(11, device=dev)
    start = gen.get_state()
    before = cuda_backend.launch_count()
    got = s.add_noise(x, t)
    launches = cuda_backend.launch_count() - before
    off = gen.get_offset()
    noise, want_off, _ = _offset_after_randn(gen, start, (3, *x.shape), dev)
    want = s.add_noise(x, t, noise=noise)
    del noise
    bad = [msg for msg in (None if off == want_off else f"generator offset {off}, torch.randn leaves {want_off}",
                           _bits_mismatch(got, want)) if msg is not None]
    assert not bad, "; ".join(bad)
    assert launches == 2


# ---- (d) generators ------------------------------------------------------------------------------------------
def _corrector_want(x, x0, mask, alpha, sigma, noise):
    """x*m + (1-m)*(alpha*x0 + sigma*noise): eager fp32 ops (one kernel each, nothing contracted), then x's dtype."""
    xf, x0f = x.float(), x0.float()
    return (xf * mask + (1 - mask) * (alpha * x0f + sigma * noise)).to(x.dtype)


def test_corrector_draws_from_its_own_generator(dev):
    import dpm_solver_b200 as new
    ns = _sched(new)
    x0, x = _data((3, 4, 160, 161), 1, dev), _data((3, 4, 160, 161), 2, dev)
    mask = torch.rand((160, 161), device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    gen = torch.Generator(device=dev)
    gen.manual_seed(20241015)
    torch.randn(9, device=dev, generator=gen)
    start = gen.get_state()
    default = torch.cuda.default_generators[dev.index]
    default_state = default.get_state()
    corr = new.DiffEditCorrector(ns, x0, mask, generator=gen)
    t = torch.tensor([0.45], device=dev)
    got = corr(x, t, 0)
    assert torch.equal(default.get_state(), default_state)        # the default generator is not touched
    off = gen.get_offset()
    noise, want_off, _ = _offset_after_randn(gen, start, (1, *x.shape), dev)
    assert off == want_off
    alpha, sigma, _ = corr._alpha_sigma(t, 0)
    _assert_same(got, _corrector_want(x, x0, mask, alpha, sigma, noise[0]))


def test_second_device_uses_its_generator_and_sm_count(cuda_backend):
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    d1 = torch.device("cuda", 1)
    G = _threads(d1)
    for T, n in ((1, 4 * G + 1), (3, G + 1)):
        bad = _raw_noise_check(cuda_backend, T, n, d1, seed=17, pre=33)
        assert not bad, f"T={T}, n={n}: " + "; ".join(bad)


# ---- (e) the corrector -----------------------------------------------------------------------------------------
def _mask(kind, shape, dev):
    """Non-binary weights (negative, above 1, exactly 0 and 1) of the given broadcast shape."""
    B, Ch, H, W = shape
    ms = {"hw": (H, W), "chw": (Ch, H, W), "11hw": (1, 1, H, W), "b1hw": (B, 1, H, W), "full": shape}[kind]
    m = _data(ms, 7, dev) * 0.8 + 0.5
    flat = m.reshape(-1)
    flat[::5] = 0.0
    flat[1::7] = 1.0
    return m


def _corrector_check(be, x, x0, mask, alpha, sigma, dev, seed, launches=1, chunk=64):
    gen = torch.cuda.default_generators[dev.index]
    torch.cuda.manual_seed(seed)
    torch.randn(13, device=dev)
    start = gen.get_state()
    before = be.launch_count()
    got = be.diffedit_corrector(x, x0, mask, alpha, sigma)
    n_launch = be.launch_count() - before
    off = gen.get_offset()
    noise, want_off, _ = _offset_after_randn(gen, start, (1, *x.shape), dev)
    bad = [] if off == want_off else [f"generator offset {off}, torch.randn leaves {want_off}"]
    noise = noise[0]
    assert got.dtype == x.dtype
    for b in range(0, x.shape[0], chunk):            # elementwise, so evaluating a slice of the batch at a time is exact
        m = mask[b:b + chunk] if mask.dim() == 4 and mask.shape[0] == x.shape[0] else mask
        msg = _bits_mismatch(got[b:b + chunk], _corrector_want(x[b:b + chunk], x0[b:b + chunk], m, alpha, sigma,
                                                               noise[b:b + chunk]))
        if msg is not None:
            bad.append(f"values (from batch row {b}): {msg}")
            break
    assert not bad, "; ".join(bad)
    assert n_launch == launches


def _alpha_sigma(t):
    import dpm_solver_b200 as new
    ns = _sched(new)
    te = torch.tensor([t], dtype=torch.float32)
    return float(ns.marginal_alpha(te)), float(ns.marginal_std(te))


_DT = [torch.float32, torch.bfloat16, torch.float16]
_DT_IDS = ["f32", "bf16", "f16"]


@pytest.mark.parametrize("shape", [(2, 4, 64, 64), (3, 3, 17, 5)])
@pytest.mark.parametrize("kind", ["hw", "chw", "11hw", "b1hw", "full"])
@pytest.mark.parametrize("dtype", _DT, ids=_DT_IDS)
def test_corrector_masks(cuda_backend, dev, dtype, kind, shape):
    """Every mask broadcast, non-binary weights, and x / x0 with non-finite, subnormal and fp16-overflowing values."""
    x = _with_specials(_data(shape, 21, dev) * 2).to(dtype)
    x0 = _with_specials(_data(shape, 22, dev) * 2).flip(-1).contiguous().to(dtype)
    alpha, sigma = _alpha_sigma(0.3)
    _corrector_check(cuda_backend, x, x0, _mask(kind, shape, dev), alpha, sigma, dev, seed=40 + len(kind))


_EDGES = {"257": lambda G: 257, "G-1": lambda G: G - 1, "G+1": lambda G: G + 1, "4G+1": lambda G: 4 * G + 1,
          "8G-1": lambda G: 8 * G - 1, "2^24+1": lambda G: (1 << 24) + 1}


@pytest.mark.parametrize("size", list(_EDGES))
@pytest.mark.parametrize("dtype", _DT, ids=_DT_IDS)
def test_corrector_sizes(cuda_backend, dev, dtype, size):
    n = _EDGES[size](_threads(dev))
    shape = (1, 1, 1, n)
    x = _with_specials(_data(shape, 23, dev)).to(dtype)
    x0 = _data(shape, 24, dev).to(dtype)
    alpha, sigma = _alpha_sigma(0.71)
    _corrector_check(cuda_backend, x, x0, _mask("hw", shape, dev), alpha, sigma, dev, seed=n % 9973)


def test_corrector_beyond_two_pow_29(cuda_backend, dev):
    """bf16 latents of 5.4e8 elements: the corrector's noise is split in two like torch.randn's."""
    shape = (2049, 4, 256, 256)
    x = _data(shape, 25, dev, torch.bfloat16)
    x0 = _data(shape, 26, dev, torch.bfloat16)
    assert x.numel() > SPLIT
    alpha, sigma = _alpha_sigma(0.55)
    _corrector_check(cuda_backend, x, x0, _mask("hw", shape, dev), alpha, sigma, dev, seed=5, launches=2)


# ---- (f) fallbacks and errors ----------------------------------------------------------------------------------
def test_seventeen_labels_take_torch_randn(dev):
    import dpm_solver_b200 as new
    s = new.DPM_Solver(None, _sched(new))
    x = _data((2, 3, 16, 16), 4, dev)
    t = torch.linspace(0.01, 0.99, 17, device=dev)
    gen = torch.cuda.default_generators[dev.index]
    torch.cuda.manual_seed(17)
    torch.randn(5, device=dev)
    start = gen.get_state()
    got = s.add_noise(x, t)
    off = gen.get_offset()
    noise, want_off, _ = _offset_after_randn(gen, start, (17, *x.shape), dev)
    assert off == want_off
    _assert_same(got, s.add_noise(x, t, noise=noise))


def test_graph_capture_takes_torch_randn(dev):
    """Under capture add_noise draws with torch.randn (graph-safe generator state); a replay equals the explicit path
    fed the randn of the generator state it replayed at."""
    import dpm_solver_b200 as new
    s = new.DPM_Solver(None, _sched(new))
    x = _data((2, 4, 32, 32), 5, dev)
    t = torch.tensor([0.2, 0.8])
    s.add_noise(x, t)                                   # warm up outside the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = s.add_noise(x, t)
    gen = torch.cuda.default_generators[dev.index]
    torch.cuda.manual_seed(99)
    torch.randn(21, device=dev)
    start = gen.get_state()
    graph.replay()
    torch.cuda.synchronize(dev)
    off = gen.get_offset()
    noise, want_off, _ = _offset_after_randn(gen, start, (2, *x.shape), dev)
    assert off == want_off
    _assert_same(static, s.add_noise(x, t, noise=noise))
    del graph


def test_capi_rejects_bad_offsets_and_label_counts(cuda_backend, dev):
    be = cuda_backend
    lib = be._lib
    x = torch.zeros(64, device=dev)
    out = torch.full((17, 64), 7.0, device=dev)
    coef = (C.c_float * 17)(*([0.5] * 17))
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

    def add_noise(t_count, offset):
        return lib.dpm_add_noise_philox(C.c_void_p(out.data_ptr()), C.c_void_p(x.data_ptr()), 64, t_count, coef, coef,
                                        123, offset, DPM_F32, DPM_F32, stream)

    assert add_noise(2, 6) == DPM_ERR_ARG
    assert b"multiple of 4" in lib.dpm_last_error()
    assert add_noise(-1, 4) < 0
    assert add_noise(17, 4) < 0
    before = be.launch_count()
    assert add_noise(0, 4) == 0                        # no labels: nothing to draw
    assert be.launch_count() == before
    torch.cuda.synchronize(dev)
    assert bool((out == 7.0).all())
    assert add_noise(16, 8) == 0
    torch.cuda.synchronize(dev)
    assert not bool((out[:16] == 7.0).any()) and bool((out[16] == 7.0).all())
    mask = torch.ones(64, device=dev)
    rc = lib.dpm_diffedit_corrector(C.c_void_p(out.data_ptr()), C.c_void_p(x.data_ptr()), C.c_void_p(x.data_ptr()),
                                    C.c_void_p(mask.data_ptr()), 64, 64, 0.5, 0.5, 123, 2, DPM_F32, stream)
    assert rc == DPM_ERR_ARG
