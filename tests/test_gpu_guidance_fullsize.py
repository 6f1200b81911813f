"""The regional-guidance, CFG++ and CFG-Zero* step kernels at sizes where their grid wraps, on the H100: [16,4,128,128]
under the default tuning and under (2,128,1) and (2,64,2), whose grids are smaller than the tile count, so that each
CTA's grid-stride loop crosses samples with real per-sample operands (maps, scales, thresholds); the generic kernels past
their grid cap on [16,3,127,129] (a per-sample size that is not a multiple of 8); dpm_cfgzero_scale at B = 64; and
sample() at [4,4,64,64] with non-trivial masks against the reference composition. Each launch is checked bit for bit
against the numpy executor on the same operands (one launch per executor call: vectorised, a few seconds each)."""
import pytest
import torch

from cfgzero_oracle import CFGZeroOracle
from oracle import ref_loader
from test_gpu_cfg_mask import _check as check_masked, _masked_args
from test_gpu_cfg_pp import _args as cfgpp_args, _check as check_cfgpp
from test_gpu_cfg_zero_star import _args as cfgzero_args, _check_step as check_cfgzero, same

pytestmark = pytest.mark.gpu
DTS = {"f32": torch.float32, "bf16": torch.bfloat16}
TUNINGS = [(2, 0, 0), (2, 128, 1), (2, 64, 2)]        # (variant, threads, CTAs per SM); 0 = the default
BIG = (16, 4, 128 * 128)                               # [16,4,128,128] as (B, C, S)
ODD = (16, 3, 127 * 129)                               # per sample 49149: the generic kernels, 786k elements
FORMS = {"LIN1": 1, "DIFF2": 4, "MS3": 5}
KINDS4 = ("pixb", "pixs", "p1b", "elb")                # per-sample pixel, shared pixel, per-sample period 1, element


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 40 * 2 ** 30


@pytest.fixture()
def tuned(cuda_backend):
    yield cuda_backend
    cuda_backend.set_tuning(2, 0, 0)


@pytest.mark.parametrize("tuning", TUNINGS, ids=lambda t: "%d-%d-%d" % t)
@pytest.mark.parametrize("sd", list(DTS))
@pytest.mark.parametrize("form", list(FORMS))
def test_masked_step_grid_wraps(tuned, form, sd, tuning):
    tuned.set_tuning(*tuning)
    gen = torch.Generator().manual_seed(FORMS[form])
    for thr in (False, True):
        a = _masked_args(FORMS[form], 0, True, DTS[sd], DTS[sd], 4, *BIG, gen, KINDS4)
        check_masked(tuned, a, thr)


@pytest.mark.parametrize("tuning", TUNINGS, ids=lambda t: "%d-%d-%d" % t)
@pytest.mark.parametrize("sd", list(DTS))
@pytest.mark.parametrize("order", [1, 2])
def test_cfgpp_step_grid_wraps(tuned, order, sd, tuning):
    tuned.set_tuning(*tuning)
    gen = torch.Generator().manual_seed(order)
    check_cfgpp(tuned, cfgpp_args(0, DTS[sd], DTS[sd], BIG[0], BIG[1] * BIG[2], gen, 1 if order == 1 else 4,
                                  per_sample=True))


@pytest.mark.parametrize("tuning", TUNINGS, ids=lambda t: "%d-%d-%d" % t)
@pytest.mark.parametrize("sd", list(DTS))
def test_cfgzero_step_grid_wraps(tuned, sd, tuning):
    tuned.set_tuning(*tuning)
    gen = torch.Generator().manual_seed(5)
    for form in (1, 4):
        check_cfgzero(tuned, cfgzero_args(4, True, DTS[sd], DTS[sd], BIG[0], BIG[1] * BIG[2], gen, form,
                                          per_sample=True))


@pytest.mark.parametrize("sd", list(DTS))
def test_generic_kernels_past_their_grid_cap(cuda_backend, sd):
    """Per-sample maps, scales and thresholds over 16 samples of 49149 elements: the generic (scalar) kernels' grid
    stops at SMs x 8 CTAs of 256 threads, so their grid-stride loop crosses samples."""
    gen = torch.Generator().manual_seed(9)
    dt = DTS[sd]
    for form in (1, 4):
        check_masked(cuda_backend, _masked_args(form, 0, True, dt, dt, 3, *ODD, gen, ("pixb", "p1b", "elb")), True)
        check_cfgpp(cuda_backend, cfgpp_args(0, dt, dt, ODD[0], ODD[1] * ODD[2], gen, form, per_sample=True))
        check_cfgzero(cuda_backend, cfgzero_args(0, True, dt, dt, ODD[0], ODD[1] * ODD[2], gen, form, per_sample=True))


@pytest.mark.parametrize("ps", [8193, 16384, 3 * 64 * 64])
def test_cfgzero_scale_at_b64(cuda_backend, ps):
    gen = torch.Generator().manual_seed(ps)
    a = cfgzero_args(0, True, torch.float32, torch.float32, 64, ps, gen)
    s = cuda_backend.cfgzero_scale(a.e_cond, a.e_uncond)
    same(s, CFGZeroOracle().cfgzero_scale(a.e_cond.cpu(), a.e_uncond.cpu()))


@pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")
@pytest.mark.parametrize("K", [2, 4])
def test_sample_fp32_masks_vs_reference(cuda_backend, K):
    """fp32 [4,4,64,64] with per-sample pixel, [B,1,1,1] and element masks (values 0, negatives, quarters): bit for bit
    the reference composition, noise/dpmsolver++ with thresholding and v/dpmsolver."""
    import dpm_solver_b200 as new
    from cases import seeded
    from test_cfg_mask import reference_composed
    from test_cfg_multi import SCALES as MULTI_SCALES, conds
    from test_cfg_rescale import inner_net, schedules
    _, _, pns = schedules("sd")
    shape = (4, 4, 64, 64)
    g = torch.Generator().manual_seed(K)
    q = lambda s: torch.randint(-4, 9, s, generator=g).float() * 0.25
    masks = [q((4, 1, 64, 64)), q((4, 1, 1, 1)), q(shape), q((4, 1, 64, 64))][:K]
    x = seeded(shape, 11)
    for mt, algo, thr in (("noise", "dpmsolver++", True), ("v", "dpmsolver", False)):
        fn = new.model_wrapper(inner_net(), pns, model_type=mt, guidance_type="classifier-free",
                               condition=[c.cuda() for c in conds(K, 4)], unconditional_condition=torch.zeros(4, 1).cuda(),
                               guidance_scale=MULTI_SCALES[K], guidance_mask=[m.cuda() for m in masks])
        skw = dict(steps=8, order=2, method="multistep", skip_type="time_uniform")
        kw = dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
        yp = new.DPM_Solver(fn, pns, **kw).sample(x.cuda(), **skw)
        ref, rns, composed = reference_composed(mt, K, MULTI_SCALES[K], masks, batch=4)
        yr = ref.DPM_Solver(composed, rns, **kw).sample(x.clone(), **skw)
        assert yp.cpu().numpy().tobytes() == yr.numpy().tobytes(), (mt, K)
