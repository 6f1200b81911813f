"""Guidance rescale on the H100: the ratio kernel against an fp64 oracle, the rescaling fused step against the numpy
executor bit for bit, and sample() end to end against the unmodified reference fed an eager-rescale network."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from cases import exact_net, make_betas, seeded
from test_cfg_rescale import PHI, S, RescaleOracle, inner_net, ratio64, ref_rescaled_net, schedules

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16"), ("bf16", "f32"), ("f16", "f32")]   # (model, state)


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def ulp_dist(a, b):
    """|a - b| in fp32 ulps for finite values of one sign; non-finite values must match exactly (NaN == NaN)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    fin = np.isfinite(a) & np.isfinite(b)
    assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~fin & ~np.isnan(a)], b[~fin & ~np.isnan(b)])
    ia = a[fin].view(np.int32).astype(np.int64)
    ib = b[fin].view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return int(np.abs(ia - ib).max()) if ia.size else 0


def halves(B, ps, dtype, gen, regime="random", offset=0):
    """(e_cond, e_uncond) of B samples of ps elements, optionally as views `offset` elements into their storage."""
    n = B * ps
    c = torch.randn(n + offset, generator=gen, dtype=torch.float64) * 2 + 0.3
    u = torch.randn(n + offset, generator=gen, dtype=torch.float64) * 1.5 - 0.1
    if regime == "large_mean":      # mean/std = 1e6 in sample 0
        c[offset:offset + ps] = 1e6 + torch.randn(ps, generator=gen, dtype=torch.float64)
        u[offset:offset + ps] = 1e6 + torch.randn(ps, generator=gen, dtype=torch.float64)
    elif regime == "special":       # constant samples, NaN and inf
        c[offset:offset + ps] = 0.5
        u[offset:offset + ps] = 0.5
        if B > 1:
            c[offset + ps] = float("nan")
        if B > 2:
            u[offset + 2 * ps] = float("inf")
        if B > 3:
            c[offset + 3 * ps:offset + 4 * ps] = u[offset + 3 * ps:offset + 4 * ps]   # g == out_u: r = std_c/std_c
    c = c.to(dtype).cuda()[offset:].reshape(B, ps)
    u = u.to(dtype).cuda()[offset:].reshape(B, ps)
    return c, u


SIZES = [1, 7, 8, 9, 8191, 8193, 3 * 256 * 256]


@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("ps", SIZES)
def test_ratio_kernel_vs_fp64(cuda_backend, dt, ps):
    gen = torch.Generator().manual_seed(ps)
    B = 5 if ps < 100000 else 3
    regimes = ["random", "special"] + (["large_mean"] if dt != "f16" else [])   # 1e6 is beyond fp16's range
    for regime in regimes:
        for offset in (0, 1):
            c, u = halves(B, ps, DT[dt], gen, regime, offset)
            r = cuda_backend.cfg_rescale_ratio(c, u, S)
            r2 = cuda_backend.cfg_rescale_ratio(c, u, S)
            assert r.cpu().numpy().tobytes() == r2.cpu().numpy().tobytes(), "ratio is not deterministic"
            cn, un = c.float().cpu().numpy(), u.float().cpu().numpy()
            want = ratio64(cn, (un + np.float32(S) * (cn - un)).astype(np.float32))
            got = r.cpu().numpy()
            assert ulp_dist(got, want) <= 2, (regime, offset, got, want)
            if ps == 1:
                assert np.isnan(got).all()
            for b in range(B):      # a sample alone (aligned, fresh storage) gives the same bits as inside the batch
                rb = cuda_backend.cfg_rescale_ratio(c[b:b + 1].clone(), u[b:b + 1].clone(), S)
                assert rb.cpu().numpy().tobytes() == got[b:b + 1].tobytes(), (regime, offset, b)


def test_ratio_kernel_channels_last(cuda_backend):
    gen = torch.Generator().manual_seed(3)
    out = torch.randn(8, 4, 24, 24, generator=gen).cuda().contiguous(memory_format=torch.channels_last)
    out[4:] = out[4:] * 1.7 + 0.2
    u, c = out.chunk(2)
    got = cuda_backend.cfg_rescale_ratio(c, u, S).cpu().numpy()
    cn, un = c.cpu().numpy(), u.cpu().numpy()
    assert ulp_dist(got, ratio64(cn, (un + np.float32(S) * (cn - un)).astype(np.float32))) <= 2


COEF = dict(a=0.9, c0=-0.3, c1=0.2, c2=0.1, w0=1.5, w1=0.7, w2=0.4, w3=0.6, w4=0.3, alpha_e=0.8, sigma_e=0.6)


def _step_args(form, param, px0, md, sd, B, ps, gen, layout="c", dev_coef=False):
    from dpm_solver_b200.ops import StepArgs
    shape = (B, 3, ps // 3) if layout == "c" else (B, 4, ps // 16, 4)

    def t(dtype, scale=1.0):
        v = (torch.randn(shape, generator=gen) * scale).to(dtype).cuda()
        return v.contiguous(memory_format=torch.channels_last) if layout == "cl" else v
    x = t(sd)
    ec, eu = t(md, 1.3), t(md)
    a = StepArgs(form=form, n_model=2, x=x if form else None, xe=x, e_cond=ec, e_uncond=eu, param=param,
                 predict_x0=px0, guidance=S, state_dtype=sd, want_m_out=True, phi=PHI,
                 m1=t(sd) if form in (2, 3, 4, 5, 6) else None, m2=t(sd) if form in (3, 5, 6) else None, **COEF)
    a.c0_on_old = form == 4 and param % 2 == 1
    if dev_coef:
        v = [COEF[k] for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e")]
        a.coef_dev = torch.tensor(v + [0.] * 5, dtype=torch.float32).cuda()
    return a


def _check_step(be, a):
    import dataclasses
    a.ratio = be.cfg_rescale_ratio(a.e_cond, a.e_uncond, a.guidance)
    a.per_sample = a.e_cond.numel() // a.e_cond.shape[0]
    m, o = be.step(a)
    cpu = lambda v: None if not torch.is_tensor(v) else v.cpu()
    ac = dataclasses.replace(a, **{f.name: cpu(getattr(a, f.name)) for f in dataclasses.fields(a)
                                   if torch.is_tensor(getattr(a, f.name))})
    ac.coef_dev = None
    mw, ow = RescaleOracle().step(ac)
    assert m.float().cpu().numpy().tobytes() == mw.float().numpy().tobytes()
    if ow is not None:
        assert o.float().cpu().numpy().tobytes() == ow.float().numpy().tobytes()


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [3 * 64, 3 * 37])      # whole packets per sample (FAST when possible) / tails
def test_rescaled_step_vs_numpy(cuda_backend, pair, ps):
    gen = torch.Generator().manual_seed(ps)
    for form in range(7):
        for param in range(4):
            for px0 in (False, True):
                _check_step(cuda_backend, _step_args(form, param, px0, DT[pair[0]], DT[pair[1]], 5, ps, gen))


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
def test_rescaled_step_channels_last_and_dev_coef(cuda_backend, pair):
    gen = torch.Generator().manual_seed(7)
    for form in range(7):
        for param in (0, 2):
            _check_step(cuda_backend, _step_args(form, param, True, DT[pair[0]], DT[pair[1]], 4, 16 * 12, gen, "cl"))
            if form:
                _check_step(cuda_backend, _step_args(form, param, True, DT[pair[0]], DT[pair[1]], 4, 3 * 40, gen,
                                                     dev_coef=True))


# ---- end to end --------------------------------------------------------------------------------------------------
SHAPE = (4, 4, 16, 16)


def _pair(model_type, algo, thr, phi=PHI):
    import dpm_solver_b200 as new
    ref, rns, pns = schedules("sd")
    B = SHAPE[0]
    uc, c = torch.zeros(B, 1), torch.ones(B, 1)
    rfn = ref.model_wrapper(ref_rescaled_net(inner_net(), uc, c, S, phi), rns, model_type=model_type)
    pfn = new.model_wrapper(inner_net(), pns, model_type=model_type, guidance_type="classifier-free",
                            condition=c.cuda(), unconditional_condition=uc.cuda(), guidance_scale=S,
                            guidance_rescale=phi)
    kw = dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
    return ref.DPM_Solver(rfn, rns, **kw), pfn, pns, kw


E2E = [(mt, m, o, al, th) for mt in ("noise", "x_start", "v", "score")
       for (m, o) in (("multistep", 2), ("multistep", 3), ("singlestep", 3), ("singlestep_fixed", 2))
       for (al, th) in (("dpmsolver", False), ("dpmsolver++", False), ("dpmsolver++", True))]


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_sample_fp32_vs_reference(cuda_backend):
    import dpm_solver_b200 as new
    x = seeded(SHAPE, 11)
    exact = 0
    for mt, method, order, algo, thr in E2E:
        rs, pfn, pns, kw = _pair(mt, algo, thr)
        skw = dict(steps=8, order=order, method=method, skip_type="time_uniform")
        yr = rs.sample(x.clone(), **skw).numpy()
        yp = new.DPM_Solver(pfn, pns, **kw).sample(x.cuda(), **skw).cpu().numpy()
        assert rel_err(yp, yr) <= 1e-5, (mt, method, order, algo, thr)
        exact += yp.tobytes() == yr.tobytes()
    print("\nfp32 sample() bitwise equal to the reference: %d of %d cases" % (exact, len(E2E)))


# max relative deviation from the fp32 reference measured on an H100 80GB HBM3 (700 W power limit) with these inputs:
# 1.11e-2 (bf16), 1.47e-3 (f16); pinned at 1.5x
BOUND_16 = {torch.bfloat16: 1.67e-2, torch.float16: 2.2e-3}


@pytest.mark.parametrize("sd", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_sample_16bit_state(cuda_backend, sd):
    import dpm_solver_b200 as new
    x = seeded(SHAPE, 11)
    worst = 0.
    for mt in ("noise", "v"):
        rs, pfn, pns, kw = _pair(mt, "dpmsolver++", False)
        skw = dict(steps=8, order=2, method="multistep", skip_type="time_uniform")
        yr = rs.sample(x.clone(), **skw).numpy()
        yp = new.DPM_Solver(pfn, pns, state_dtype=sd, **kw).sample(x.cuda(), **skw).float().cpu().numpy()
        worst = max(worst, rel_err(yp, yr))
    print("\n%s state: max rel err %.3g" % (sd, worst))
    assert worst <= BOUND_16[sd]


def test_capture_replays_bit_identically(cuda_backend):
    import dpm_solver_b200 as new
    _, pfn, pns, kw = _pair("noise", "dpmsolver++", False)
    s = new.DPM_Solver(pfn, pns, **kw)
    x = seeded(SHAPE, 2).cuda()
    skw = dict(steps=6, order=2, method="multistep")
    eager = s.sample(x.clone(), **skw)
    g = s.capture(x, **skw)
    y1 = g(x).clone()
    y2 = g(x).clone()
    assert torch.equal(y1, y2) and torch.equal(y1, eager)


def test_device_controller_adaptive_matches_host(cuda_backend, monkeypatch, capsys):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import DPM_Solver
    _, pfn, pns, kw = _pair("noise", "dpmsolver", False)
    x = seeded(SHAPE, 4).cuda()
    y_dev = new.DPM_Solver(pfn, pns, **kw).sample(x, order=2, method="adaptive", atol=0.05, rtol=0.1)
    nfe_dev = int(capsys.readouterr().out.split()[-1])
    monkeypatch.setattr(DPM_Solver, "adaptive_controller", "host")
    y_host = new.DPM_Solver(pfn, pns, **kw).sample(x, order=2, method="adaptive", atol=0.05, rtol=0.1)
    nfe_host = int(capsys.readouterr().out.split()[-1])
    assert nfe_dev == nfe_host
    assert rel_err(y_dev.cpu().numpy(), y_host.cpu().numpy()) <= 1e-4


@pytest.mark.parametrize("method,order", [("multistep", 3), ("singlestep", 3)])
def test_phi_change_is_not_served_by_a_stale_launch(cuda_backend, method, order):
    import dpm_solver_b200 as new
    _, pfn, pns, kw = _pair("noise", "dpmsolver++", False, phi=0.)
    x = seeded(SHAPE, 6).cuda()
    skw = dict(steps=6, order=order, method=method)
    s = new.DPM_Solver(pfn, pns, **kw)
    y0 = s.sample(x, **skw)
    y0b = s.sample(x, **skw)           # the prepared launches of the phi = 0 run now exist
    pfn.guidance_rescale = PHI
    y1 = s.sample(x, **skw)
    _, fresh_fn, _, _ = _pair("noise", "dpmsolver++", False)
    y_fresh = new.DPM_Solver(fresh_fn, pns, **kw).sample(x, **skw)
    assert torch.equal(y0, y0b) and not torch.equal(y1, y0)
    assert torch.equal(y1, y_fresh)


def _worker(rank, world, port, outdir):
    for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper
    from dpm_solver_b200.distributed import shard_batch
    ns = NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    x = shard_batch(seeded((12, 3, 16, 16), 5)).contiguous().cuda()
    b = x.shape[0]
    fn = model_wrapper(inner_net(), ns, guidance_type="classifier-free", condition=torch.ones(b, 1).cuda(),
                       unconditional_condition=torch.zeros(b, 1).cuda(), guidance_scale=S, guidance_rescale=PHI)
    y = DPM_Solver(fn, ns, plan_broadcast=True).sample(x, steps=8, order=3)
    np.save(os.path.join(outdir, f"y{rank}.npy"), y.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_nccl_shards_equal_single_gpu(tmp_path, cuda_backend):
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper
    world = min(torch.cuda.device_count(), 4)
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    ns = NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    fn = model_wrapper(inner_net(), ns, guidance_type="classifier-free", condition=torch.ones(12, 1).cuda(),
                       unconditional_condition=torch.zeros(12, 1).cuda(), guidance_scale=S, guidance_rescale=PHI)
    full = DPM_Solver(fn, ns).sample(seeded((12, 3, 16, 16), 5).cuda(), steps=8, order=3)
    got = np.concatenate([np.load(tmp_path / f"y{r}.npy") for r in range(world)])
    np.testing.assert_array_equal(got, full.cpu().numpy())
