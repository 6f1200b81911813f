"""Per-sample classifier-free guidance on the H100: the guided fused step and the guided ratio pass against the numpy
executor and fp64 bit for bit, and sample() end to end against the unmodified reference run once per distinct scale."""
import dataclasses
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from cases import make_betas, seeded
from test_cfg_per_sample import SCALES, GuidedOracle, reference_rows, rowwise_net
from test_cfg_rescale import PHI, inner_net, ratio64, schedules
from test_gpu_cfg_rescale import COEF, DT, PAIRS, _step_args, halves, rel_err, ulp_dist

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def _scales(B):
    return torch.tensor([SCALES[b % len(SCALES)] for b in range(B)], dtype=torch.float32).cuda()


def _offset(t, k=1):
    """t as a view k elements into a fresh storage (unaligned for the vector kernels)."""
    buf = torch.empty(t.numel() + k, dtype=t.dtype, device=t.device)
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


def _check_step(be, a, rescale, thr):
    B = a.e_cond.shape[0]
    a.per_sample = a.e_cond.numel() // B
    a.guidance_b = _scales(B)
    a.ratio = be.cfg_rescale_ratio(a.e_cond, a.e_uncond, a.guidance_b) if rescale else None
    if thr:
        a.thr = (torch.rand(B, generator=torch.Generator().manual_seed(B)) * 2 + 0.5).cuda()
    m, o = be.step(a)
    cpu = lambda v: None if not torch.is_tensor(v) else v.cpu()
    ac = dataclasses.replace(a, **{f.name: cpu(getattr(a, f.name)) for f in dataclasses.fields(a)
                                   if torch.is_tensor(getattr(a, f.name))})
    ac.coef_dev = None
    mw, ow = GuidedOracle().step(ac)
    assert m.float().cpu().numpy().tobytes() == mw.float().numpy().tobytes()
    if ow is not None:
        assert o.float().cpu().numpy().tobytes() == ow.float().numpy().tobytes()


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [3 * 64, 3 * 37])      # whole packets per sample (FAST when possible) / tails
@pytest.mark.parametrize("rescale", [False, True])
def test_guided_step_vs_numpy(cuda_backend, pair, ps, rescale):
    gen = torch.Generator().manual_seed(ps)
    for form in range(7):
        for param in range(4):
            for px0 in (False, True):
                for thr in ((False, True) if px0 else (False,)):
                    a = _step_args(form, param, px0, DT[pair[0]], DT[pair[1]], 7, ps, gen)
                    _check_step(cuda_backend, a, rescale, thr)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("rescale", [False, True])
def test_guided_step_views_channels_last_and_dev_coef(cuda_backend, pair, rescale):
    gen = torch.Generator().manual_seed(7)
    md, sd = DT[pair[0]], DT[pair[1]]
    for form in range(7):
        for param in (0, 2):
            _check_step(cuda_backend, _step_args(form, param, True, md, sd, 6, 16 * 12, gen, "cl"), rescale, True)
            a = _step_args(form, param, True, md, sd, 6, 3 * 40, gen)
            a.e_cond, a.e_uncond = _offset(a.e_cond), _offset(a.e_uncond)      # views offset by one element
            _check_step(cuda_backend, a, rescale, param == 0)
            if form:
                _check_step(cuda_backend, _step_args(form, param, True, md, sd, 6, 3 * 40, gen, dev_coef=True),
                            rescale, False)


@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("ps", [1, 9, 8192, 8193, 3 * 64 * 64])
def test_guided_ratio_vs_fp64_and_per_sample_scalar(cuda_backend, dt, ps):
    gen = torch.Generator().manual_seed(ps)
    B = 6
    for offset in (0, 1):
        c, u = halves(B, ps, DT[dt], gen, "random", offset)
        s = _scales(B)
        got = cuda_backend.cfg_rescale_ratio(c, u, s).cpu().numpy()
        cn, un = c.float().cpu().numpy(), u.float().cpu().numpy()
        sn = s.cpu().numpy().reshape(-1, 1)
        assert ulp_dist(got, ratio64(cn, (un + sn * (cn - un)).astype(np.float32))) <= 2
        for b in range(B):
            one = cuda_backend.cfg_rescale_ratio(c, u, float(s[b])).cpu().numpy()
            assert got[b:b + 1].tobytes() == one[b:b + 1].tobytes(), (offset, b)


# ---- end to end --------------------------------------------------------------------------------------------------
SHAPE = (len(SCALES), 4, 16, 16)


def _product_fn(model_type, scales, phi, B=SHAPE[0]):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    fn = new.model_wrapper(inner_net(), pns, model_type=model_type, guidance_type="classifier-free",
                           condition=torch.ones(B, 1).cuda(), unconditional_condition=torch.zeros(B, 1).cuda(),
                           guidance_scale=scales, guidance_rescale=phi)
    return fn, pns


E2E = [(mt, m, o, al, th, phi) for mt in ("noise", "x_start", "v", "score")
       for (m, o) in (("multistep", 2), ("singlestep", 3), ("singlestep_fixed", 2))
       for (al, th) in (("dpmsolver", False), ("dpmsolver++", False), ("dpmsolver++", True))
       for phi in (0., PHI)]


def test_sample_fp32_vs_reference(cuda_backend):
    import dpm_solver_b200 as new
    x = seeded(SHAPE, 11)
    bad = []
    for mt, method, order, algo, thr, phi in E2E:
        fn, pns = _product_fn(mt, torch.tensor(SCALES).cuda(), phi)
        kw = dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
        skw = dict(steps=8, order=order, method=method, skip_type="time_uniform")
        yp = new.DPM_Solver(fn, pns, **kw).sample(x.cuda(), **skw).cpu().numpy()
        for rows, yr in reference_rows(mt, algo, thr, phi, lambda s, xr: s.sample(xr, **skw), x):
            if yp[rows].tobytes() != yr.numpy().tobytes():
                bad.append((mt, method, order, algo, thr, phi, rows, rel_err(yp[rows], yr.numpy())))
    print("\nfp32 sample() rows bitwise equal to the reference: %d of %d cases" % (len(E2E) - len(bad), len(E2E)))
    assert not bad, bad


@pytest.mark.parametrize("sd", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("thr,phi", [(False, 0.), (True, 0.), (True, PHI)])
def test_sample_16bit_state_vs_executor(cuda_backend, sd, thr, phi):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    x = seeded(SHAPE, 11)
    kw = dict(algorithm_type="dpmsolver++", correcting_x0_fn="dynamic_thresholding" if thr else None, state_dtype=sd)
    skw = dict(steps=8, order=3, method="singlestep", skip_type="time_uniform")
    for mt in ("noise", "v"):
        fn, pns = _product_fn(mt, torch.tensor(SCALES).cuda(), phi)
        yp = new.DPM_Solver(fn, pns, **kw).sample(x.cuda(), **skw).float().cpu().numpy()
        old = ops._backend
        ops.set_backend(GuidedOracle())
        try:
            import dpm_solver_b200 as new2
            _, _, pns_cpu = schedules("sd")
            fn_cpu = new2.model_wrapper(inner_net(), pns_cpu, model_type=mt, guidance_type="classifier-free",
                                        condition=torch.ones(SHAPE[0], 1), unconditional_condition=torch.zeros(SHAPE[0], 1),
                                        guidance_scale=torch.tensor(SCALES), guidance_rescale=phi)
            yw = new2.DPM_Solver(fn_cpu, pns_cpu, **kw).sample(x.clone(), **skw).float().numpy()
        finally:
            ops.set_backend(old)
        assert yp.tobytes() == yw.tobytes(), (mt, rel_err(yp, yw))


def test_capture_picks_up_new_scales(cuda_backend):
    import dpm_solver_b200 as new
    scales = torch.tensor(SCALES).cuda()
    fn, pns = _product_fn("noise", scales, PHI)
    s = new.DPM_Solver(fn, pns, correcting_x0_fn="dynamic_thresholding")
    x = seeded(SHAPE, 2).cuda()
    skw = dict(steps=6, order=2, method="multistep")
    g = s.capture(x, **skw)
    y1 = g(x).clone()
    assert torch.equal(y1, s.sample(x.clone(), **skw))
    scales.copy_(torch.tensor([2.0, 3.0, 1.0, -1.0, 0.0, 9.0]))      # written in place between replays
    y2 = g(x).clone()
    fresh_fn, _ = _product_fn("noise", torch.tensor([2.0, 3.0, 1.0, -1.0, 0.0, 9.0]).cuda(), PHI)
    want = new.DPM_Solver(fresh_fn, pns, correcting_x0_fn="dynamic_thresholding").sample(x.clone(), **skw)
    assert not torch.equal(y1, y2) and torch.equal(y2, want)


@pytest.mark.parametrize("phi", [0., PHI])
def test_device_controller_adaptive_matches_host(cuda_backend, monkeypatch, capsys, phi):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import DPM_Solver
    fn, pns = _product_fn("v", torch.tensor(SCALES).cuda(), phi)
    x = seeded(SHAPE, 4).cuda()
    y_dev = new.DPM_Solver(fn, pns, correcting_x0_fn="dynamic_thresholding").sample(
        x, order=2, method="adaptive", atol=0.05, rtol=0.1)
    nfe_dev = int(capsys.readouterr().out.split()[-1])
    monkeypatch.setattr(DPM_Solver, "adaptive_controller", "host")
    y_host = new.DPM_Solver(fn, pns, correcting_x0_fn="dynamic_thresholding").sample(
        x, order=2, method="adaptive", atol=0.05, rtol=0.1)
    nfe_host = int(capsys.readouterr().out.split()[-1])
    assert nfe_dev == nfe_host
    assert rel_err(y_dev.cpu().numpy(), y_host.cpu().numpy()) <= 1e-4


@pytest.mark.parametrize("model_type,phi", [("noise", 0.), ("noise", PHI), ("v", PHI)])
@pytest.mark.parametrize("algo,thr", [("dpmsolver", False), ("dpmsolver++", False), ("dpmsolver++", True)])
def test_adaptive_vs_reference_with_rowwise_net(cuda_backend, capsys, model_type, phi, algo, thr):
    """The GPU run (device controller where it applies) against the unmodified reference fed the per-row combine:
    the same NFE, 1e-5 relative."""
    import dpm_solver_b200 as new
    from unittest import mock
    ref, rns, _ = schedules("sd")
    x = seeded(SHAPE, 11)
    kw = dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
    akw = dict(order=2, method="adaptive", atol=0.05, rtol=0.1)
    rs = ref.DPM_Solver(ref.model_wrapper(rowwise_net(SCALES, phi), rns, model_type=model_type), rns, **kw)
    with mock.patch("builtins.print") as pr:
        yr = rs.sample(x.clone(), **akw).numpy()
        nfe_r = pr.call_args[0][-1]
    fn, pns = _product_fn(model_type, torch.tensor(SCALES).cuda(), phi)
    capsys.readouterr()
    yp = new.DPM_Solver(fn, pns, **kw).sample(x.cuda(), **akw).cpu().numpy()
    nfe_p = int(capsys.readouterr().out.split()[-1])
    assert nfe_p == nfe_r
    assert rel_err(yp, yr) <= 1e-5, rel_err(yp, yr)


def test_full_size_rows_equal_scalar_runs(cuda_backend):
    """The c3 shape in bf16: every row of a mixed-scale run equals that row of the one-scale run with its scale."""
    import dpm_solver_b200 as new
    B = 2048
    ns = new.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, 4, 64, 64, generator=gen, device="cuda").to(torch.bfloat16)
    vals = [7.5, 1.0, 3.0, 12.0]
    scales = torch.tensor([vals[b % 4] for b in range(B)], dtype=torch.float32, device="cuda")
    net = lambda xi, t, c: (xi.float() * 0.9 - 0.1 * c.reshape(-1, 1, 1, 1)).to(xi.dtype)

    def run(s):
        fn = new.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B, 1, device="cuda"),
                               unconditional_condition=torch.zeros(B, 1, device="cuda"), guidance_scale=s)
        return new.DPM_Solver(fn, ns, state_dtype=torch.bfloat16).sample(x, steps=15, order=3, method="singlestep")
    y = run(scales)
    for i, v in enumerate(vals):
        assert torch.equal(y[i::4], run(v)[i::4]), v


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
    s = shard_batch(torch.tensor(SCALES * 2)).contiguous().cuda()
    b = x.shape[0]
    fn = model_wrapper(inner_net(), ns, guidance_type="classifier-free", condition=torch.ones(b, 1).cuda(),
                       unconditional_condition=torch.zeros(b, 1).cuda(), guidance_scale=s, guidance_rescale=PHI)
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
                       unconditional_condition=torch.zeros(12, 1).cuda(), guidance_scale=torch.tensor(SCALES * 2).cuda(),
                       guidance_rescale=PHI)
    full = DPM_Solver(fn, ns).sample(seeded((12, 3, 16, 16), 5).cuda(), steps=8, order=3)
    got = np.concatenate([np.load(tmp_path / f"y{r}.npy") for r in range(world)])
    np.testing.assert_array_equal(got, full.cpu().numpy())
