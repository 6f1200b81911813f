"""Paths beside the sampling loop, against the UNMODIFIED reference (oracle/_ref): classifier guidance (:315-321),
`add_noise` (:1012-1030), the 'cosine' schedule of the older vendored copies (SD dpm_solver.py:114-175), NaN
propagation of dynamic thresholding (:416-425), and the ADVICE.md round-1 corner cases. Each test runs on the numpy
executor (CPU) and on CudaBackend (`-m gpu`); the reference arm always runs on CPU."""
import numpy as np
import pytest
import torch

from cases import exact_net, make_betas, seeded
from helpers import rel_err
from oracle import ref_loader

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="oracle/_ref not built and no reference tree")
EXECUTORS = ["numpy-executor", pytest.param("cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=EXECUTORS)
def dev(request):
    from dpm_solver_b200 import ops
    old = ops._backend
    if request.param == "cuda":
        ops.set_backend(ops.CudaBackend())
        yield "cuda:0"
    else:
        from oracle_backend import OracleBackend
        ops.set_backend(OracleBackend())
        yield "cpu"
    ops.set_backend(old)


def _sched(mod, name="sd"):
    kind, betas = make_betas(name)
    return mod.NoiseScheduleVP("linear") if kind == "linear" else mod.NoiseScheduleVP("discrete", betas=torch.from_numpy(betas))


# ---- classifier guidance -----------------------------------------------------------------------------
def _classifier_fn(x, t_input, y, **kw):
    """log p(y|x) whose gradient is exact on every device: quadratic in x with power-of-two weights."""
    w = (y.to(x.dtype) * 0.125 + 0.25).reshape(-1, 1, 1, 1)
    return (w * x * x * 0.5 + 0.0625 * x).sum(dim=(1, 2, 3)) + t_input * 0.001


@pytest.mark.parametrize("model_type", ["noise", "x_start", "v", "score"])
@pytest.mark.parametrize("algo,order,method", [("dpmsolver++", 2, "multistep"), ("dpmsolver", 3, "singlestep")])
def test_classifier_guidance_sample(dev, model_type, algo, order, method):
    """model_fn's classifier branch inside sample(): noise - scale * sigma_t * grad (:315-321), bit-identical."""
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    B = 3
    x = seeded((B, 3, 8, 8), 77)
    outs = []
    for mod, d in ((ref, "cpu"), (new, dev)):
        ns = _sched(mod, "ddpm_linear")
        y = torch.tensor([1, 4, 7], device=d)
        fn = mod.model_wrapper(exact_net, ns, model_type=model_type, guidance_type="classifier", condition=y,
                               guidance_scale=2.5, classifier_fn=_classifier_fn)
        s = mod.DPM_Solver(fn, ns, algorithm_type=algo)
        outs.append(s.sample(x.to(d), steps=9, order=order, method=method).cpu())
    assert torch.isfinite(outs[0]).all()
    np.testing.assert_array_equal(outs[1].numpy(), outs[0].numpy())


def test_classifier_guidance_direct_call_per_sample_times(dev):
    """model_fn(x, t) called directly with a different time label per sample."""
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    x = seeded((4, 3, 8, 8), 5)
    t = torch.tensor([0.9, 0.5, 0.25, 0.05])
    outs = []
    for mod, d in ((ref, "cpu"), (new, dev)):
        ns = _sched(mod, "sd")
        fn = mod.model_wrapper(exact_net, ns, model_type="v", guidance_type="classifier",
                               condition=torch.tensor([0, 1, 2, 3], device=d), guidance_scale=1.5, classifier_fn=_classifier_fn)
        outs.append(fn(x.to(d), t.to(d)).cpu())
    np.testing.assert_array_equal(outs[1].numpy(), outs[0].numpy())


# ---- add_noise -----------------------------------------------------------------------------------------
def test_add_noise_golden_and_reference(dev, golden):
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    g = golden["glue"]
    x, noise = torch.from_numpy(g["x"]), torch.from_numpy(g["add_noise_in"])
    ns = _sched(new, "sd")
    got = new.DPM_Solver(None, ns).add_noise(x.to(dev), torch.tensor([0.3, 0.8], device=dev), noise=noise.to(dev))
    np.testing.assert_array_equal(got.cpu().numpy(), g["add_noise"])
    # single time label -> [B, ...] (squeeze rule :1027-1030); 16-bit input promotes like the reference
    for dt in (torch.float32, torch.bfloat16):
        xr = seeded((2, 4, 8, 8), 3).to(dt)
        nz = seeded((1, 2, 4, 8, 8), 4).to(dt)
        want = ref.DPM_Solver(None, _sched(ref, "sd")).add_noise(xr, torch.tensor([0.45]), noise=nz)
        have = new.DPM_Solver(None, ns).add_noise(xr.to(dev), torch.tensor([0.45], device=dev), noise=nz.to(dev))
        assert have.shape == want.shape
        np.testing.assert_array_equal(have.float().cpu().numpy(), want.float().numpy())


@pytest.mark.parametrize("sdt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("xdt", [torch.float32, "state"])
def test_add_noise_16bit_state_rounds_once(dev, sdt, xdt):
    """A 16-bit state with fp32 noise: the reference's fp32 result rounded once to the state dtype, not a sum of
    noise already rounded to 16 bits."""
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    x = seeded((2, 4, 8, 8), 3).to(sdt if xdt == "state" else xdt)
    nz = seeded((2, 2, 4, 8, 8), 4)
    t = torch.tensor([0.3, 0.8])
    want = ref.DPM_Solver(None, _sched(ref, "sd")).add_noise(x, t, noise=nz).to(sdt)
    have = new.DPM_Solver(None, _sched(new, "sd"), state_dtype=sdt).add_noise(x.to(dev), t.to(dev), noise=nz.to(dev))
    assert have.dtype == sdt and have.shape == want.shape
    np.testing.assert_array_equal(have.float().cpu().numpy(), want.float().numpy())


# ---- 'cosine' schedule of the older vendored copies -----------------------------------------------------
def test_cosine_schedule_scalars_match_vendored_copy():
    """NoiseScheduleVP('cosine') (examples/stable-diffusion/.../dpm_solver.py:114-175): every marginal and the inverse."""
    from dpm_solver_b200 import NoiseScheduleVP
    old = ref_loader.load("sd_dpm_solver")
    a, b = NoiseScheduleVP("cosine"), old.NoiseScheduleVP("cosine")
    assert a.T == b.T == 0.9946 and a.total_N == b.total_N
    t = torch.cat([torch.linspace(1e-3, 0.9946, 257), torch.tensor([1e-5, 0.5, 0.9946])])
    for name in ("marginal_log_mean_coeff", "marginal_alpha", "marginal_std", "marginal_lambda"):
        np.testing.assert_array_equal(getattr(a, name)(t).numpy(), getattr(b, name)(t).numpy(), err_msg=name)
    lam = b.marginal_lambda(t)
    np.testing.assert_array_equal(a.inverse_lambda(lam).numpy(), b.inverse_lambda(lam).numpy())


@pytest.mark.parametrize("kw", [dict(steps=12, order=2, method="multistep", skip_type="time_uniform"),
                                dict(steps=10, order=3, method="singlestep", skip_type="logSNR")])
def test_cosine_schedule_sample_matches_vendored_copy(dev, kw):
    """A whole sample() on the cosine schedule against the vendored copy that defines it."""
    import dpm_solver_b200 as new
    old = ref_loader.load("sd_dpm_solver")
    x = seeded((2, 3, 8, 8), 31)
    net = lambda xx, tt: 0.1 * xx + ((tt * 0.05) - 0.02).reshape(-1, 1, 1, 1)
    outs = []
    for mod, d in ((old, "cpu"), (new, dev)):
        ns = mod.NoiseScheduleVP("cosine")
        s = mod.DPM_Solver(mod.model_wrapper(net, ns), ns, algorithm_type="dpmsolver++")
        outs.append(s.sample(x.to(d), t_end=1e-3, **kw).cpu())
    assert torch.isfinite(outs[0]).all()
    np.testing.assert_array_equal(outs[1].numpy(), outs[0].numpy())


# ---- NaN propagation (ADVICE r1) ----------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(3, 3, 16, 16), (3, 3, 64, 64)])     # cluster kernel / streaming pipeline
def test_dynamic_thresholding_propagates_nan(dev, shape):
    """A NaN in one sample: torch.quantile returns NaN for that sample, clamp and division propagate it (:422-424);
    the other samples are untouched."""
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    x0 = seeded(shape, 9) * 2.0
    x0[1, 0, 2, 3] = float("nan")
    want = ref.DPM_Solver(None, _sched(ref)).dynamic_thresholding_fn(x0, None)
    have = new.DPM_Solver(None, _sched(new)).dynamic_thresholding_fn(x0.to(dev), None).cpu()
    assert torch.isnan(want[1]).all() and torch.isfinite(want[0]).all()
    np.testing.assert_array_equal(have.numpy(), want.numpy())      # NaNs compare equal positionally


@pytest.mark.parametrize("ratio", [0.995, 0.997, 1.0])
@pytest.mark.parametrize("shape", [(3, 3, 16, 16), (3, 3, 64, 64)])     # cluster kernel / streaming pipeline
def test_dynamic_thresholding_infinite_order_statistics(dev, shape, ratio):
    """+-inf in x0 reaches the quantile's order statistics. With pos = fl(ratio*(n-1)), lo = floor(pos), w = pos - lo
    and k infinities in a sample of n: k = n - lo puts both order statistics at inf (inf - inf in the lerp: NaN),
    k = n - lo - 1 puts only the upper one there (fma(w, inf, lo) = inf for w < 0.5, fma(w-1, inf, inf) = NaN for
    w >= 0.5), k = n - lo - 2 leaves both finite. ratio 0.995 gives w = 0.165 (n = 768) and 0.565 (n = 12288), 0.997
    gives 0.70 and 0.14, 1.0 gives w = 0 with lo = n - 1, where a single inf is already inf - inf. The quantile
    becomes NaN or inf, torch.maximum keeps a NaN, and clamp / division spread it over the sample (:422-424)."""
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    B, n = shape[0], int(np.prod(shape[1:]))
    pos = np.float32(ratio) * np.float32(n - 1)
    lo = int(np.floor(pos))
    x0 = (seeded(shape, 9) * 2.0).reshape(B, n)
    rs = np.random.RandomState(n)
    for b, k in enumerate((n - lo - 2, n - lo, n - lo - 1)):
        k = max(k, 1)
        idx = torch.from_numpy(rs.permutation(n)[:k])
        x0[b, idx] = torch.from_numpy(np.where(rs.rand(k) < 0.5, np.inf, -np.inf).astype(np.float32))
    x0 = x0.reshape(shape)
    want = ref.DPM_Solver(None, _sched(ref), dynamic_thresholding_ratio=ratio).dynamic_thresholding_fn(x0, None)
    have = new.DPM_Solver(None, _sched(new), dynamic_thresholding_ratio=ratio).dynamic_thresholding_fn(x0.to(dev), None).cpu()
    assert torch.isnan(want[1]).all()                              # both order statistics infinite
    if ratio < 1.0:
        assert torch.isfinite(want[0]).all()
    np.testing.assert_array_equal(have.numpy(), want.numpy())      # NaNs compare equal positionally


def test_adaptive_raises_on_nan_error_estimate(dev):
    """The reference would spin forever on a NaN error estimate (:1002-1008); the product raises."""
    import dpm_solver_b200 as new
    ns = _sched(new, "vp_linear")
    s = new.DPM_Solver(new.model_wrapper(lambda x, t: x * float("nan"), ns), ns, algorithm_type="dpmsolver")
    with pytest.raises(FloatingPointError):
        s.sample(seeded((2, 3, 8, 8), 1).to(dev), method="adaptive", order=2, t_end=1e-3)


# ---- corner cases from ADVICE.md (round 1) ---------------------------------------------------------------------
def test_cfg_on_channels_last_input(dev):
    """out2 = x_in[B:] of a channels_last doubled batch is dense but not `is_contiguous()`."""
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    B = 2
    x = seeded((B, 4, 8, 8), 13)
    outs = []
    for mod, d, cl in ((ref, "cpu", False), (new, dev, True)):
        ns = _sched(mod)
        net = lambda xx, tt, cc: exact_net(xx, tt) + 0.05 * cc.reshape(-1, 1, 1, 1)
        fn = mod.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B, 1, device=d),
                               unconditional_condition=torch.zeros(B, 1, device=d), guidance_scale=4.0)
        xi = x.to(d)
        if cl:
            xi = xi.contiguous(memory_format=torch.channels_last)
        outs.append(mod.DPM_Solver(fn, ns).sample(xi, steps=8, order=2).cpu())
    np.testing.assert_array_equal(outs[1].contiguous().numpy(), outs[0].numpy())


def test_fp32_network_output_with_16bit_state_and_thresholding(dev):
    """model fp32 -> state bf16 with dynamic thresholding: quantile and step take the same dtype mix."""
    import dpm_solver_b200 as new
    ns = _sched(new, "ddpm_linear")
    net = lambda xx, tt: exact_net(xx.float(), tt)
    s = new.DPM_Solver(new.model_wrapper(net, ns), ns, correcting_x0_fn="dynamic_thresholding", state_dtype=torch.bfloat16)
    x = seeded((2, 3, 64, 64), 17).to(dev)
    y = s.sample(x, steps=8, order=2)
    assert y.dtype == torch.bfloat16 and torch.isfinite(y.float()).all()
    ref = ref_loader.load("dpm_solver_pytorch")
    nr = _sched(ref, "ddpm_linear")
    yr = ref.DPM_Solver(ref.model_wrapper(net, nr), nr, correcting_x0_fn="dynamic_thresholding").sample(x.cpu().bfloat16().float(), steps=8, order=2)
    assert rel_err(y.float().cpu().numpy(), yr.numpy()) < 0.06


@pytest.mark.gpu
def test_capture_with_denoise_to_zero(cuda_backend):
    """The denoise tail (:1236-1238) uses cached device tables: the whole run stays CUDA-graph capturable."""
    import dpm_solver_b200 as new
    ns = _sched(new)
    s = new.DPM_Solver(new.model_wrapper(exact_net, ns), ns)
    x = seeded((2, 4, 16, 16), 1234).cuda()
    kw = dict(steps=10, order=2, denoise_to_zero=True)
    eager = s.sample(x, **kw)
    run = s.capture(x, **kw)
    assert torch.equal(run(x), eager)
    ref = ref_loader.load("dpm_solver_pytorch")
    nr = _sched(ref)
    yr = ref.DPM_Solver(ref.model_wrapper(exact_net, nr), nr).sample(x.cpu(), **kw)
    np.testing.assert_array_equal(eager.cpu().numpy(), yr.numpy())


# ---- in-kernel noise: add_noise(noise=None) and the DiffEdit corrector (SURVEY 8f-3) ------------------------------
def _notebook_corrector(sampler, init_latent, mask):
    """diffedit_inpaint.ipynb, `corrector_fn`, verbatim."""
    def corrector_fn(x, t, step):
        ratio = sampler.time_to_ratio(t)
        stochastic_intermediate = sampler.stochastic_encode(init_latent, ratio)
        x = x * mask + (1 - mask) * stochastic_intermediate
        return x
    return corrector_fn


def test_diffedit_corrector_matches_the_notebook_on_the_host_executor(oracle_backend):
    """DiffEditCorrector == the notebook's corrector_fn on top of the unmodified SD adapter, same CPU generator state."""
    import adapters as A
    import dpm_solver_b200 as new
    mod = A.load_sd_adapter(A.reference_solver("sd"), "diffedit_ref", "cpu")
    sampler = mod.DPMSolverSampler(A.StubLatentDiffusion("cpu"))
    x0, x = seeded((1, 4, 16, 16), 3), seeded((1, 4, 16, 16), 4)
    mask = (seeded((16, 16), 5) > 0).float()
    ns = new.NoiseScheduleVP("discrete", alphas_cumprod=sampler.alphas_cumprod)
    fused = new.DiffEditCorrector(ns, x0, mask, time_fn=lambda t: sampler.ratio_to_time(sampler.time_to_ratio(t)))
    ref_fn = _notebook_corrector(sampler, x0, mask)
    for step, tv in enumerate([0.9, 0.5, 0.05]):
        t = torch.tensor(tv)
        torch.manual_seed(100 + step)
        want = ref_fn(x, t, step)
        torch.manual_seed(100 + step)
        got = fused(x, t, step)
        np.testing.assert_array_equal(got.numpy(), want.numpy())


def test_diffedit_corrector_reused_with_other_times_on_the_host_executor(oracle_backend):
    """One corrector called again with the same step numbers at other times (another `steps` or `t_end` of the solver
    holding it), then with another `time_fn`: (alpha, sigma) follow the time, never the step number."""
    import adapters as A
    import dpm_solver_b200 as new
    mod = A.load_sd_adapter(A.reference_solver("sd"), "diffedit_ref", "cpu")
    sampler = mod.DPMSolverSampler(A.StubLatentDiffusion("cpu"))
    x0, x = seeded((1, 4, 16, 16), 3), seeded((1, 4, 16, 16), 4)
    mask = (seeded((16, 16), 5) > 0).float()
    ns = new.NoiseScheduleVP("discrete", alphas_cumprod=sampler.alphas_cumprod)
    fused = new.DiffEditCorrector(ns, x0, mask, time_fn=lambda t: sampler.ratio_to_time(sampler.time_to_ratio(t)))
    ref_fn = _notebook_corrector(sampler, x0, mask)
    labels = [torch.tensor(v) for v in (0.9, 0.5, 0.05, 0.8, 0.3, 0.02)]      # kept alive, as a solver's tables are
    for n, t in enumerate(labels + labels):
        torch.manual_seed(200 + n)
        want = ref_fn(x, t, n % 3)
        torch.manual_seed(200 + n)
        np.testing.assert_array_equal(fused(x, t, n % 3).numpy(), want.numpy())
    fused.time_fn = None                    # the same label and step again, re-noised to the label's own level now
    te = labels[1].reshape(1)
    torch.manual_seed(300)
    inter = ns.marginal_alpha(te) * x0 + ns.marginal_std(te) * torch.randn((1, *x0.shape))[0]
    torch.manual_seed(300)
    np.testing.assert_array_equal(fused(x, labels[1], 1).numpy(), (x * mask + (1 - mask) * inter).numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("shape,times", [((2, 4, 64, 64), [0.5]), ((3, 3, 17, 5), [0.3, 0.8, 0.05]), ((700, 4, 64, 64), [0.6])])
def test_add_noise_draws_torch_randn_in_the_kernel(cuda_backend, shape, times):
    """add_noise(noise=None): the noise is generated in registers by curand's Philox exactly as torch.randn would
    have (same seed and offset -> same normals, generator advanced identically), then alpha*x + sigma*noise."""
    import dpm_solver_b200 as new
    s = new.DPM_Solver(None, _sched(new))
    x = seeded(shape, 8).cuda()
    t = torch.tensor(times, device="cuda")
    torch.manual_seed(1234)
    torch.randn(5, device="cuda")                                     # a non-zero philox offset
    state = torch.cuda.get_rng_state()
    before = cuda_backend.launch_count()
    got = s.add_noise(x, t)
    assert cuda_backend.launch_count() == before + 1                  # ONE launch, no randn kernel, no noise tensor
    after_fused = torch.cuda.default_generators[0].get_offset()
    torch.cuda.set_rng_state(state)
    noise = torch.randn((len(times), *x.shape), device="cuda")       # what the reference draws (:1024)
    assert torch.cuda.default_generators[0].get_offset() == after_fused
    want = s.add_noise(x, t, noise=noise)                             # explicit-noise path (bit-exact vs the reference)
    assert got.shape == want.shape
    assert torch.equal(got, want)
    ref = ref_loader.load("dpm_solver_pytorch")
    want_cpu = ref.DPM_Solver(None, _sched(ref)).add_noise(x.cpu(), t.cpu(), noise=noise.cpu())
    np.testing.assert_array_equal(got.cpu().numpy(), want_cpu.numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("sdt", [torch.float32, torch.bfloat16])
def test_diffedit_corrector_fused_kernel(cuda_backend, sdt):
    """One launch == x*mask + (1-mask)*(alpha*x0 + sigma*randn) with torch's own normals for the generator state."""
    import dpm_solver_b200 as new
    ns = _sched(new)
    x0, x = seeded((2, 4, 64, 64), 3).cuda().to(sdt), seeded((2, 4, 64, 64), 4).cuda().to(sdt)
    mask = (seeded((64, 64), 5) > 0).float().cuda()
    fused = new.DiffEditCorrector(ns, x0, mask)
    t = torch.tensor([0.4], device="cuda")
    torch.manual_seed(77)
    state = torch.cuda.get_rng_state()
    before = cuda_backend.launch_count()
    got = fused(x, t, 0)
    assert cuda_backend.launch_count() == before + 1
    torch.cuda.set_rng_state(state)
    noise = torch.randn((1, *x0.shape), device="cuda")
    te = t.cpu().to(sdt).float()            # stochastic_encode rebuilds the label in the latent's dtype (sampler.py:94)
    al, sg = float(ns.marginal_alpha(te)), float(ns.marginal_std(te))
    inter = (torch.tensor(al) * x0.float().cpu() + torch.tensor(sg) * noise[0].cpu())
    want = x.float().cpu() * mask.cpu() + (1 - mask.cpu()) * inter
    np.testing.assert_array_equal(got.float().cpu().numpy(), want.to(sdt).float().numpy())
