"""TCFG and frequency-decoupled guidance at full size on the H100.

FDG: dpm_fdg_guided bit for bit against fdg_oracle.fdg_exact in fp32, bf16 and fp16, with shared and per-sample scales,
at [16, 4, H, W] on planes that reach each of k_fdg_guided's three CTA shapes (at most 512, 1024 and 2048 packets of 8
per plane), its opt-in past 48 KiB of shared memory, its scalar loads (H*W % 8 != 0, strided planes), odd coarse
levels, extreme aspect ratios and the smallest planes; 64 x 64 also 5-D, 126 x 130 also channels_last and transposed.
sample() at [4, 16, 128, 128] with 5 levels of per-sample scales against the unmodified reference, and bf16 network
outputs at [16, 4, 128, 128] against the numpy executor.

TCFG: dpm_tcfg_words at B = 64; the TCFG step at [16, 4, 128, 128] under the default tuning, (2, 128, 1) and (2, 64, 2),
whose grids are smaller than the tile count, so that each CTA's grid-stride loop crosses samples with per-sample words
and scales, and the generic kernel at [16, 3, 127, 129]; sample() at [4, 4, 64, 64] with thresholding against the
unmodified reference."""
import pytest
import torch

from fdg_oracle import FDGOracle, fdg_exact
from oracle import ref_loader
from tcfg_oracle import TCFGOracle
from test_gpu_cfg_zero_star import _args as step_args, same
from test_gpu_fdg import net as fdg_net, on, pair, same_bits, scale_rows, solve
from test_gpu_tcfg import _check_step as check_tcfg_step, net as tcfg_net

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTS = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
TUNINGS = [(2, 0, 0), (2, 128, 1), (2, 64, 2)]        # (variant, threads, CTAs per SM); 0 = the default
BIG = (16, 4, 128 * 128)
ODD = (16, 3, 127 * 129)
needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")

# (plane, levels): the path each reaches
PLANES = [((64, 64), 5),        # CTA shape 0 at its top (512 packets)
          ((72, 64), 4),        # shape 1
          ((64, 128), 5),       # shape 1 past 48 KiB of shared memory (49.6 KB)
          ((128, 64), 5),       # likewise (50.2 KB)
          ((96, 88), 4),        # shape 2
          ((126, 130), 2),      # shape 2, scalar loads, an odd coarse level (63 x 65)
          ((127, 129), 1),      # no pyramid, scalar loads
          ((6, 2730), 2),       # extreme aspect ratios: about 98 and 120 KB of shared memory
          ((2730, 6), 2),
          ((6, 6), 2),          # the smallest planes
          ((3, 3), 1)]


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 40 * 2 ** 30


@pytest.fixture()
def tuned(cuda_backend):
    yield cuda_backend
    cuda_backend.set_tuning(2, 0, 0)


def _check_fdg(be, c, u, scales, levels):
    sc = scales.to(DEV) if torch.is_tensor(scales) else scales
    got = be.fdg_guided(c, u, sc, levels)
    assert got.dtype == c.dtype and got.shape == c.shape
    assert same_bits(got, fdg_exact(c.cpu(), u.cpu(), scales, levels))
    return got


# ---- dpm_fdg_guided ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", list(DTS))
@pytest.mark.parametrize("hw,levels", PLANES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_fdg_planes(cuda_backend, hw, levels, dt):
    c, u = pair(hw[0] * 7 + hw[1], (16, 4) + hw, DTS[dt])
    c, u = c.to(DEV), u.to(DEV)
    for scales in ([9.0, 4.5, 2.0, -1.0, 3.0][:levels], scale_rows(levels, 16, levels)):
        _check_fdg(cuda_backend, c, u, scales, levels)


@pytest.mark.parametrize("dt", list(DTS))
def test_fdg_5d_and_strided_planes(cuda_backend, dt):
    c, u = pair(21, (2, 3, 4, 64, 64), DTS[dt])
    _check_fdg(cuda_backend, c.to(DEV), u.to(DEV), scale_rows(5, 2, 21), 5)
    c, u = pair(22, (16, 4, 126, 130), DTS[dt])
    rows = scale_rows(2, 16, 22)
    cl = lambda t: t.to(DEV).contiguous(memory_format=torch.channels_last)
    got = _check_fdg(cuda_backend, cl(c), cl(u), rows, 2)
    assert got.is_contiguous(memory_format=torch.channels_last)
    # transposed views: planes whose rows are strided
    tr = lambda t: t.transpose(-1, -2).contiguous().to(DEV).transpose(-1, -2)
    _check_fdg(cuda_backend, tr(c), tr(u), rows, 2)
    _check_fdg(cuda_backend, tr(c), u.to(DEV), [5.0, 1.5], 2)


# ---- FDG sample() ----------------------------------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("mt,thr", [("noise", True), ("flow", False)])
def test_fdg_sample_fp32_vs_reference(cuda_backend, mt, thr):
    """fp32 [4, 16, 128, 128], 5 levels of per-sample scales: bit for bit the unmodified reference driving a network that
    returns the FDG output (fdg_oracle.guided_net)."""
    from fdg_oracle import guided_net
    from test_fdg import reference_schedule
    ref = ref_loader.load("dpm_solver_pytorch")
    shape = (4, 16, 128, 128)
    rows = torch.tensor([[7.0, 3.5, 1.5, 1.0, 2.0], [2.0, 4.0, 1.0, 0.0, -1.0], [1.0, 1.0, 1.0, 1.0, 1.0],
                         [10.0, 2.5, 7.0, 3.5, 1.5]])
    skw = dict(steps=5, order=2, method="multistep")
    y = solve(DEV, mt=mt, scales=rows, shape=shape, thr=thr, skw=skw, calls=1)[0].cpu()
    rns = reference_schedule(mt)
    g = guided_net(fdg_net, torch.zeros(4, 1), torch.ones(4, 1), rows)
    if mt == "flow":
        from flow_oracle import reference_solver
        rs = reference_solver(g, rns, "dpmsolver++", thresholding=thr)
    else:
        rs = ref.DPM_Solver(ref.model_wrapper(g, rns, model_type=mt), rns, algorithm_type="dpmsolver++",
                            correcting_x0_fn="dynamic_thresholding" if thr else None)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(0))
    yr = rs.sample(x, **skw)
    assert torch.equal(y, yr), float((y - yr).abs().max())


def test_fdg_sample_bf16_outputs_vs_executor(cuda_backend):
    """bf16 network outputs (fp32 state) at [16, 4, 128, 128], 4 levels of shared scales: bit for bit the executor."""
    def bf16_net(x, t, c):
        return fdg_net(x, t, c).to(torch.bfloat16)
    kw = dict(scales=(8.0, 4.0, 2.0, 1.0), shape=(16, 4, 128, 128), model=bf16_net, skw=dict(steps=4, order=2), calls=1)
    got = solve(DEV, **kw)[0]
    want = on(FDGOracle(), lambda: solve("cpu", **kw))[0]
    assert torch.equal(got.cpu(), want), float((got.cpu() - want).abs().max())


# ---- TCFG ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ps", [8193, 16384, 3 * 64 * 64])
def test_tcfg_words_at_b64(cuda_backend, ps):
    gen = torch.Generator().manual_seed(ps)
    a = step_args(0, True, torch.float32, torch.float32, 64, ps, gen)
    same(cuda_backend.tcfg_words(a.e_cond, a.e_uncond), TCFGOracle().tcfg_words(a.e_cond.cpu(), a.e_uncond.cpu()))


@pytest.mark.parametrize("tuning", TUNINGS, ids=lambda t: "%d-%d-%d" % t)
@pytest.mark.parametrize("sd", ["f32", "bf16"])
def test_tcfg_step_grid_wraps(tuned, sd, tuning):
    tuned.set_tuning(*tuning)
    gen = torch.Generator().manual_seed(6)
    for form in (1, 4):
        check_tcfg_step(tuned, step_args(4, True, DTS[sd], DTS[sd], BIG[0], BIG[1] * BIG[2], gen, form,
                                         per_sample=True))


@pytest.mark.parametrize("sd", ["f32", "bf16"])
def test_tcfg_generic_kernel_past_its_grid_cap(cuda_backend, sd):
    gen = torch.Generator().manual_seed(10)
    for form in (1, 4):
        check_tcfg_step(cuda_backend, step_args(0, True, DTS[sd], DTS[sd], ODD[0], ODD[1] * ODD[2], gen, form,
                                                per_sample=True))


@needs_ref
def test_tcfg_sample_fp32_vs_reference(cuda_backend):
    """fp32 [4, 4, 64, 64], per-sample scales with a row at 1, dynamic thresholding: bit for bit the unmodified
    reference driving a network that returns the TCFG output (tcfg_oracle.guided_net)."""
    import dpm_solver_b200 as new
    from tcfg_oracle import guided_net
    from test_tcfg import product_schedule, reference_schedule
    ref = ref_loader.load("dpm_solver_pytorch")
    shape = (4, 4, 64, 64)
    w = torch.tensor([7.5, 1.0, 3.5, 2.0])
    x = torch.randn(shape, generator=torch.Generator().manual_seed(3))
    ns = product_schedule("noise")
    fn = new.model_wrapper(tcfg_net, ns, guidance_type="classifier-free", condition=torch.ones(4, 1, device=DEV),
                           unconditional_condition=torch.zeros(4, 1, device=DEV), guidance_scale=w.to(DEV), tcfg=True)
    skw = dict(steps=6, order=2, method="multistep")
    kw = dict(algorithm_type="dpmsolver++", correcting_x0_fn="dynamic_thresholding")
    y = new.DPM_Solver(fn, ns, **kw).sample(x.to(DEV), **skw).cpu()
    rns = reference_schedule("noise")
    g = guided_net(tcfg_net, torch.zeros(4, 1), torch.ones(4, 1), w)
    yr = ref.DPM_Solver(ref.model_wrapper(g, rns, model_type="noise"), rns, **kw).sample(x.clone(), **skw)
    assert torch.equal(y, yr), float((y - yr).abs().max())
