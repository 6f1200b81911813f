"""dpm_solver_adaptive (:956-1010): same NFE and the same sample as the reference. The error estimate
is a reduction (its summation order differs between torch-CPU, numpy and the CUDA kernel), so the
sample is compared with the north-star tolerance instead of bit for bit; the accept/reject decisions
-- hence the NFE the reference prints -- must be identical."""
import numpy as np
import pytest
import torch

from cases import exact_net, make_betas, seeded
from helpers import product_schedule, rel_err

CASES = [
    dict(name="ad23_eps_vp", schedule="vp_linear", algo="dpmsolver", order=3, t_end=1e-3, solver_type="dpmsolver"),
    dict(name="ad12_eps_vp", schedule="vp_linear", algo="dpmsolver", order=2, t_end=1e-3, solver_type="dpmsolver"),
    dict(name="ad23_pp_sd", schedule="sd", algo="dpmsolver++", order=3, t_end=None, solver_type="taylor"),
    dict(name="ad12_pp_sd", schedule="sd", algo="dpmsolver++", order=2, t_end=None, solver_type="dpmsolver"),
]


def run(c, device, capsys):
    from dpm_solver_b200 import DPM_Solver, model_wrapper
    ns = product_schedule(c["schedule"])
    x = seeded((2, 3, 8, 8), 77).to(device)
    s = DPM_Solver(model_wrapper(exact_net, ns), ns, algorithm_type=c["algo"])
    y = s.sample(x, method="adaptive", order=c["order"], t_end=c["t_end"], solver_type=c["solver_type"])
    nfe = int(capsys.readouterr().out.split()[-1])
    return y, nfe


@pytest.fixture(scope="module")
def gold():
    import os
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "adaptive.npz"))


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_adaptive_host_logic(gold, oracle_backend, capsys, c):
    y, nfe = run(c, "cpu", capsys)
    assert nfe == int(gold[c["name"] + "/nfe"])
    assert rel_err(y.numpy(), gold[c["name"] + "/y"]) <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_adaptive_gpu(gold, cuda_backend, capsys, monkeypatch, c):
    """Default (device controller): its scalars are correctly rounded fp32 (fp64 evaluation, one rounding), the host's
    SLEEF results differ from that in the last ulp of a few arguments, and an adaptive solve amplifies an ulp through
    h = theta*h*E^(-1/order): same decisions and NFE, the sample within 1e-4 -- on 40 random configurations it is
    bit-identical to the reference's CPU run in 27 and within 5e-5 in the rest, while the reference's own CUDA run
    strays up to 3e-2 and changes NFE once (tools/adaptive_probe.py, H100). Host controller: the north-star 1e-5."""
    from dpm_solver_b200 import DPM_Solver
    y, nfe = run(c, "cuda:0", capsys)
    assert nfe == int(gold[c["name"] + "/nfe"])
    assert rel_err(y.cpu().numpy(), gold[c["name"] + "/y"]) <= 1e-4
    monkeypatch.setattr(DPM_Solver, "adaptive_controller", "host")
    y, nfe = run(c, "cuda:0", capsys)
    assert nfe == int(gold[c["name"] + "/nfe"])
    assert rel_err(y.cpu().numpy(), gold[c["name"] + "/y"]) <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("shape,dt", [((5, 3, 64, 64), torch.float32), ((3, 1001), torch.float32), ((4, 4, 64, 64), torch.bfloat16)])
def test_error_norm_kernel(cuda_backend, shape, dt):
    g = torch.Generator().manual_seed(5)
    xh, xl, xp = (torch.randn(shape, generator=g).to(dt) for _ in range(3))
    xl = (xh.float() + 0.01 * xl.float()).to(dt)
    got = float(cuda_backend.error_norm(xh.cuda(), xl.cuda(), xp.cuda(), 0.0078, 0.05).cpu())
    h, l, p = (t.double().numpy() for t in (xh, xl, xp))
    delta = np.maximum(0.0078, 0.05 * np.maximum(np.abs(l), np.abs(p)))
    ref = np.sqrt(np.mean(np.square(((h - l) / delta).reshape(shape[0], -1)), axis=-1)).max()
    assert abs(got - ref) <= 2e-6 * ref


# Relative error of the kernel's E against float64 on the same (widened) inputs, from its accumulation order
# (csrc/adaptive.cu). Each term v^2, v = (h - l) / max(atol, rtol*max(|l|, |p|)), carries 4 fp32 roundings (rtol*m,
# h - l, the division, the square): 7 units of u = 2^-24 in v^2. The sum of non-negative terms then gains at most one
# u per addition on its path: a per-thread fp32 sum of <= 32 terms (31), a 5-level warp shuffle tree (5) and a
# sequential sum of 8 warp partials (7); the fp64 sum across chunks adds nothing at this scale. The mean is rounded
# to fp32 (1) and sqrtf rounds once more (1 in E); sqrt halves the relative error of the sum. The batch maximum
# keeps the bound. 10 % on top covers the second-order terms.
_U = 2.0 ** -24
ERR_NORM_RTOL = 1.1 * ((7 + 31 + 5 + 7 + 1) / 2 + 1) * _U        # 1.7e-6


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_error_norm_kernel_fuzz(cuda_backend, seed):
    """dpm_adaptive_error against float64 on random batches: f32 / bf16 / f16, B from 1 to 1000 (beyond the 256
    threads of k_err_final), per_sample around the 8192-element chunk and the 8-element packet, misaligned views (the
    scalar path), both tolerance settings, and the regimes E = 0, NaN, inf and 0/0. Non-finite results must match
    exactly, finite ones within ERR_NORM_RTOL; two calls on one input give the same bits."""
    import random
    rng = random.Random(700 + seed)
    for case in range(12):
        dt = rng.choice([torch.float32, torch.bfloat16, torch.float16])
        B = rng.choice([1, rng.randint(2, 16), rng.randint(257, 1000)])
        ps = rng.choice([1, 7, 8, rng.randint(8191, 8193), 8 * rng.randint(2, 1 << 17)])
        if rng.random() < 0.1:
            ps = 1 << 20
        B = min(B, max(1, (1 << 22) // ps))                       # at most 4 M elements per case
        off = rng.choice([0, 0, 1, 3])                             # element offset: 1, 3 take the scalar path
        atol, rtol = rng.choice([(0.0078, 0.05), (0.0, 0.05)])
        regime = rng.choice(["random", "random", "equal", "nan", "inf", "zeros"])
        n = B * ps
        g = torch.Generator().manual_seed(rng.randint(0, 1 << 30))
        xh = torch.randn(n + off, generator=g) * rng.choice([0.1, 1.0, 30.0])
        xl = xh + 0.01 * torch.randn(n + off, generator=g)
        xp = torch.randn(n + off, generator=g)
        b = rng.randrange(B)
        at = off + b * ps + rng.randrange(ps)
        if regime == "equal":
            xl = xh.clone()
        elif regime == "nan":
            rng.choice([xh, xl, xp])[at] = float("nan")
        elif regime == "inf":
            xh[at] = float("inf")
        elif regime == "zeros":
            atol = 0.0
            for t in (xh, xl, xp):
                t[off + b * ps: off + (b + 1) * ps] = 0.0
        xh, xl, xp = (t.to(dt) for t in (xh, xl, xp))
        dev = [t.cuda()[off:].view(B, ps) for t in (xh, xl, xp)]
        got = cuda_backend.error_norm(*dev, atol, rtol)
        again = cuda_backend.error_norm(*dev, atol, rtol)
        got, again = got.cpu().numpy(), again.cpu().numpy()
        assert got.tobytes() == again.tobytes(), "error norm is not deterministic"
        h, l, p = (t[off:].double().numpy().reshape(B, ps) for t in (xh, xl, xp))
        with np.errstate(all="ignore"):
            delta = np.maximum(np.float64(np.float32(atol)), np.float64(np.float32(rtol)) * np.maximum(np.abs(l), np.abs(p)))
            ref = np.sqrt(np.mean(np.square((h - l) / delta), axis=-1))
        ref = np.float64(np.nan) if np.isnan(ref).any() else ref.max()   # torch .max(): NaN wins
        e = float(got[0])
        desc = dict(seed=seed, case=case, dt=dt, B=B, ps=ps, off=off, atol=atol, rtol=rtol, regime=regime, got=e, ref=ref)
        if not np.isfinite(ref):
            assert (np.isnan(e) and np.isnan(ref)) or e == ref, desc
            continue
        assert abs(e - ref) <= ERR_NORM_RTOL * ref, desc
        if regime == "equal":
            assert e == 0.0, desc


# ---- the controller on the device (csrc/adaptive_ctl.cu) ------------------------------------------------------------
def _adaptive_cfgs(n, seed):
    import random
    from test_random_configs_vs_reference import draw_wide
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        c = draw_wide(rng)
        c.update(method="adaptive", order=rng.choice([2, 3]), atol=rng.choice([0.0078, 0.05]), rtol=rng.choice([0.05, 0.2]),
                 thresholding=False, denoise_to_zero=False)
        if c["schedule"] == "iddpm_cosine":
            continue
        out.append(c)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", range(4))
def test_device_controller_matches_reference(cuda_backend, chunk):
    """Random adaptive configurations (schedules, both algorithms and solver types, all parameterisations, CFG,
    t_start / t_end, batch shapes): the device-side controller takes the accept/reject decisions of the UNMODIFIED
    reference (same NFE) and lands on its sample within the reduction-order / device-libm tolerance."""
    import contextlib
    import io
    import dpm_solver_b200 as new
    from oracle import ref_loader
    from test_random_configs_vs_reference import run_wide
    if not ref_loader.available():
        pytest.skip("oracle/_ref not built")
    ref = ref_loader.load("dpm_solver_pytorch")

    class OnGpu:        # run_wide() builds CPU tensors: move the product arm to the device
        NoiseScheduleVP = new.NoiseScheduleVP

        @staticmethod
        def model_wrapper(net, ns, **kw):
            kw = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw.items()}
            return new.model_wrapper(net, ns, **kw)

        class DPM_Solver(new.DPM_Solver):
            def sample(self, x, **kw):
                return super().sample(x.cuda(), **kw).cpu()

    from unittest import mock
    seen_device = 0
    for c in _adaptive_cfgs(10, 9000 + chunk):
        with mock.patch("builtins.print") as pr:           # both print 'adaptive solver nfe', N (:1009)
            yr, _, _ = run_wide(ref, c)
        nfe_r = pr.call_args[0][-1]
        if not torch.isfinite(yr).all():
            continue
        before = cuda_backend.launch_count()
        with mock.patch("builtins.print") as pn:
            yn, _, _ = run_wide(OnGpu, c)
        seen_device += cuda_backend.launch_count() > before
        assert pn.call_args[0][-1] == nfe_r, ("NFE", c)
        assert rel_err(yn.numpy(), yr.numpy()) <= 2e-4, c      # measured: 0 .. 5e-5 (profiles/r02_adaptive_probe.txt)
    assert seen_device


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_device_controller_syncs_once_per_chunk(gold, cuda_backend, capsys, monkeypatch, c):
    """The only device->host read of the adaptive loop is AdaptiveController.read(): once per `adaptive_chunk`
    iterations. Same NFE and sample as the host controller (the reference's per-iteration decision)."""
    from dpm_solver_b200 import DPM_Solver, model_wrapper, ops
    reads = []
    orig = ops.AdaptiveController.read

    def counting(self):
        r = orig(self)
        reads.append(r)
        return r
    monkeypatch.setattr(ops.AdaptiveController, "read", counting)
    y_dev, nfe_dev = run(c, "cuda:0", capsys)
    iters = reads[-1][2]
    assert len(reads) == -(-iters // DPM_Solver.adaptive_chunk) and reads[-1][0] == 1
    assert nfe_dev == int(gold[c["name"] + "/nfe"]) == iters * c["order"]
    monkeypatch.setattr(DPM_Solver, "adaptive_controller", "host")
    y_host, nfe_host = run(c, "cuda:0", capsys)
    assert nfe_host == nfe_dev
    assert rel_err(y_dev.cpu().numpy(), y_host.cpu().numpy()) <= 1e-4
