"""Multi-condition classifier-free guidance on the H100: dpm_step_multi and dpm_replicate against the numpy executor and
torch.cat bit for bit, and sample() end to end against the reference composition evaluated on the CPU."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from cases import seeded
from test_cfg_multi import SCALES, MultiOracle, conds, reference
from test_cfg_rescale import inner_net, schedules
from refcheck import rms_rel_err
from test_gpu_cfg_rescale import COEF, DT, PAIRS, rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def _offset(t, k=1):
    """t as a view k elements into a fresh storage (unaligned for the vector kernels)."""
    buf = torch.empty(t.numel() + k, dtype=t.dtype, device=t.device)
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


def _multi_args(form, param, px0, md, sd, K, B, ps, gen, layout="c", dev_coef=False):
    from dpm_solver_b200.ops import StepArgs
    shape = (B, 3, ps // 3) if layout == "c" else (B, 4, ps // 16, 4)

    def t(dtype, scale=1.0, shift=0.0):
        v = (torch.randn(shape, generator=gen) * scale + shift).to(dtype).cuda()
        return v.contiguous(memory_format=torch.channels_last) if layout == "cl" else v
    x = t(sd)
    ecs = tuple(t(md, 1.0 + 0.2 * k, 0.1 * k) for k in range(K))
    a = StepArgs(form=form, n_model=2, x=x if form else None, xe=x, e_cond=ecs[0], e_uncond=t(md), e_conds=ecs,
                 scales=tuple(SCALES[K]), param=param, predict_x0=px0, state_dtype=sd, want_m_out=True,
                 m1=t(sd) if form in (2, 3, 4, 5, 6) else None, m2=t(sd) if form in (3, 5, 6) else None, **COEF)
    a.c0_on_old = form == 4 and param % 2 == 1
    if form:
        a.replicas = tuple(torch.full_like(x, float("nan")) for _ in range(K))
    if dev_coef:
        v = [COEF[k] for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e")]
        a.coef_dev = torch.tensor(v + [0.] * 5, dtype=torch.float32).cuda()
    return a


def _check(be, a, thr):
    B = a.e_cond.shape[0]
    if thr:
        a.per_sample = a.e_cond.numel() // B
        a.thr = (torch.rand(B, generator=torch.Generator().manual_seed(B)) * 2 + 0.5).cuda()
    m, o = be.step(a)
    cpu = lambda v: v.cpu() if torch.is_tensor(v) else (tuple(e.cpu() for e in v) if isinstance(v, tuple) and v and
                                                          torch.is_tensor(v[0]) else v)
    ac = dataclasses.replace(a, **{f.name: cpu(getattr(a, f.name)) for f in dataclasses.fields(a)})
    ac.coef_dev, ac.replicas = None, None
    mw, ow = MultiOracle().step(ac)
    assert m.float().cpu().numpy().tobytes() == mw.float().numpy().tobytes()
    if ow is not None:
        ob = o.float().cpu().numpy().tobytes()
        assert ob == ow.float().numpy().tobytes()
        for r in a.replicas:
            assert r.float().cpu().numpy().tobytes() == ob


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [3 * 64, 3 * 37])      # whole packets per sample (FAST when possible) / tails
@pytest.mark.parametrize("K", [2, 3, 4])
def test_step_multi_vs_executor(cuda_backend, pair, ps, K):
    gen = torch.Generator().manual_seed(ps + K)
    for form in range(7):
        for param in range(4):
            for px0 in (False, True):
                for thr in ((False, True) if px0 else (False,)):
                    _check(cuda_backend, _multi_args(form, param, px0, DT[pair[0]], DT[pair[1]], K, 5, ps, gen), thr)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("K", [2, 4])
def test_step_multi_views_channels_last_and_dev_coef(cuda_backend, pair, K):
    gen = torch.Generator().manual_seed(7 + K)
    md, sd = DT[pair[0]], DT[pair[1]]
    for form in range(7):
        for param in (0, 2):
            _check(cuda_backend, _multi_args(form, param, True, md, sd, K, 4, 16 * 12, gen, "cl"), True)
            a = _multi_args(form, param, True, md, sd, K, 4, 3 * 40, gen)
            a.e_conds = tuple(_offset(e) for e in a.e_conds)      # views offset by one element
            a.e_cond, a.e_uncond = a.e_conds[0], _offset(a.e_uncond)
            _check(cuda_backend, a, param == 0)
            if form:
                _check(cuda_backend, _multi_args(form, param, True, md, sd, K, 4, 3 * 40, gen, dev_coef=True), False)


@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
def test_replicate_equals_cat(cuda_backend, dt):
    gen = torch.Generator().manual_seed(1)
    for shape in ((3, 4, 8, 8), (5, 3, 7, 3), (1, 1)):
        x = torch.randn(shape, generator=gen).to(DT[dt]).cuda()
        for xv in (x, _offset(x)):
            for copies in (1, 2, 3, 5):
                got = cuda_backend.replicate(xv, copies)
                assert got.cpu().view(torch.uint8).numpy().tobytes() == \
                    torch.cat([xv] * copies).cpu().view(torch.uint8).numpy().tobytes()
    xc = torch.randn(2, 4, 6, 6, generator=gen).to(DT[dt]).cuda().contiguous(memory_format=torch.channels_last)
    got = cuda_backend.replicate(xc, 3)
    assert got.is_contiguous(memory_format=torch.channels_last) and torch.equal(got, torch.cat([xc] * 3))


def test_capi_argument_errors_launch_nothing(cuda_backend):
    from dpm_solver_b200 import _lib
    L = _lib.lib()
    n = 64
    t = [torch.zeros(n, device="cuda") for _ in range(8)]
    d = _lib.StepDesc()
    d.x, d.xe, d.e_uncond, d.out, d.m1 = (v.data_ptr() for v in t[:5])
    d.n, d.state_dtype, d.model_dtype, d.form, d.n_model, d.a, d.c0 = n, 0, 0, 1, 2, 1.0, 1.0
    ec = (C.c_void_p * 4)(*[v.data_ptr() for v in t[4:8]])
    sc = (C.c_float * 4)(1.0, 2.0, 3.0, 4.0)
    rp = (C.c_void_p * 4)(*[v.data_ptr() for v in t[4:8]])
    before = L.dpm_launch_count()
    for n_cond in (0, 1, 5, -1):
        assert L.dpm_step_multi(C.byref(d), ec, sc, n_cond, rp, None) == -1
    d.raw_round = 1
    assert L.dpm_step_multi(C.byref(d), ec, sc, 2, None, None) == -1
    d.raw_round = 0
    assert L.dpm_step_multi(C.byref(d), None, sc, 2, None, None) == -1
    assert L.dpm_step_multi(C.byref(d), ec, None, 2, None, None) == -1
    assert L.dpm_step_multi(C.byref(d), (C.c_void_p * 2)(t[5].data_ptr(), None), sc, 2, None, None) == -1
    assert L.dpm_step_multi(C.byref(d), ec, sc, 2, (C.c_void_p * 2)(t[6].data_ptr(), None), None) == -1
    d.out = None
    assert L.dpm_step_multi(C.byref(d), ec, sc, 2, None, None) == -1
    assert L.dpm_replicate(None, t[0].data_ptr(), n, 2, 0, None) == -1
    assert L.dpm_replicate(t[1].data_ptr(), t[0].data_ptr(), n, 0, 0, None) == -1
    torch.cuda.synchronize()
    assert L.dpm_launch_count() == before


# ---- end to end --------------------------------------------------------------------------------------------------
SHAPE = (3, 4, 16, 16)
B = SHAPE[0]


def _product(model_type, K, algo, thr, sd=None):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    fn = new.model_wrapper(inner_net(), pns, model_type=model_type, guidance_type="classifier-free",
                           condition=[c.cuda() for c in conds(K)], unconditional_condition=torch.zeros(B, 1).cuda(),
                           guidance_scale=SCALES[K])
    return new.DPM_Solver(fn, pns, algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None,
                          state_dtype=sd)


ALGOS3 = (("dpmsolver", False), ("dpmsolver++", False), ("dpmsolver++", True))
E2E = [(mt, m, o, al, th, K) for mt in ("noise", "x_start", "v", "score")
       for (m, o) in (("multistep", 2), ("singlestep", 3), ("singlestep_fixed", 2))
       for (al, th) in ALGOS3 for K in (2, 3, 4)]


def test_sample_fp32_vs_reference_composition(cuda_backend):
    x = seeded(SHAPE, 11)
    bad = []
    for mt, method, order, algo, thr, K in E2E:
        skw = dict(steps=8, order=order, method=method, skip_type="time_uniform")
        yp = _product(mt, K, algo, thr).sample(x.cuda(), **skw).cpu().numpy()
        yr = reference(mt, algo, thr, K, SCALES[K]).sample(x.clone(), **skw).numpy()
        if yp.tobytes() != yr.tobytes():
            bad.append((mt, method, order, algo, thr, K, rel_err(yp, yr)))
    print("\nfp32 sample() bitwise equal to the reference composition: %d of %d cases" % (len(E2E) - len(bad), len(E2E)))
    assert not bad, bad


@pytest.mark.parametrize("thr", [False, True])
def test_sample_bf16_state_vs_executor_and_fp32(cuda_backend, thr):
    """bf16 state: bitwise equal to the executor's bf16 run, and close to the fp32 run."""
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    x = seeded(SHAPE, 11)
    skw = dict(steps=8, order=3, method="singlestep", skip_type="time_uniform")
    for mt, K in (("noise", 2), ("v", 4)):
        y16 = _product(mt, K, "dpmsolver++", thr, torch.bfloat16).sample(x.cuda(), **skw).float().cpu().numpy()
        y32 = _product(mt, K, "dpmsolver++", thr).sample(x.cuda(), **skw).cpu().numpy()
        old = ops._backend
        ops.set_backend(MultiOracle())
        try:
            _, _, pns = schedules("sd")
            fn = new.model_wrapper(inner_net(), pns, model_type=mt, guidance_type="classifier-free", condition=conds(K),
                                   unconditional_condition=torch.zeros(B, 1), guidance_scale=SCALES[K])
            yw = new.DPM_Solver(fn, pns, algorithm_type="dpmsolver++", state_dtype=torch.bfloat16,
                                correcting_x0_fn="dynamic_thresholding" if thr else None).sample(
                x.clone(), **skw).float().numpy()
        finally:
            ops.set_backend(old)
        assert y16.tobytes() == yw.tobytes(), (mt, rel_err(y16, yw))
        assert rel_err(y16, y32) <= 5e-2 and rms_rel_err(y16, y32) <= 1e-2, (rel_err(y16, y32), rms_rel_err(y16, y32))


@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("K", [2, 3, 4])
def test_adaptive_device_controller(cuda_backend, capsys, K, algo):
    """The device controller: bitwise equal to the library's own run on the same eager-composed network with
    guidance_type="uncond" (both share the error reduction and the controller), and the reference's NFE."""
    import dpm_solver_b200 as new
    from unittest import mock
    x = seeded(SHAPE, 4)
    akw = dict(order=2, method="adaptive", atol=0.05, rtol=0.1)
    capsys.readouterr()
    y = _product("noise", K, algo, False).sample(x.cuda(), **akw)
    nfe = int(capsys.readouterr().out.split()[-1])
    inner, n = inner_net(), K + 1
    c_in = torch.cat([torch.zeros(B, 1)] + conds(K)).cuda()

    def eager(xx, t_input):
        outs = inner(torch.cat([xx] * n), torch.cat([t_input] * n), c_in).chunk(n)
        e = outs[0]
        for s, ek in zip(SCALES[K], outs[1:]):
            e = e + s * (ek - outs[0])
        return e
    _, _, pns = schedules("sd")
    y_u = new.DPM_Solver(new.model_wrapper(eager, pns, guidance_type="uncond"), pns, algorithm_type=algo).sample(
        x.cuda(), **akw)
    nfe_u = int(capsys.readouterr().out.split()[-1])
    assert nfe == nfe_u and torch.equal(y, y_u)
    with mock.patch("builtins.print") as pr:
        reference("noise", algo, False, K, SCALES[K]).sample(x.clone(), **akw)
        assert pr.call_args[0][-1] == nfe


@pytest.mark.parametrize("thr", [False, True])
def test_capture_equals_eager(cuda_backend, thr):
    s = _product("noise", 3, "dpmsolver++", thr)
    x = seeded(SHAPE, 2).cuda()
    skw = dict(steps=6, order=2, method="multistep")
    g = s.capture(x, **skw)
    assert torch.equal(g(x).clone(), s.sample(x.clone(), **skw))


@pytest.mark.parametrize("thr", [False, True])
@pytest.mark.parametrize("K", [2, 4])
def test_launch_counts(cuda_backend, K, thr):
    """Per evaluation: one fused launch; with thresholding one materialising launch and the quantile's launches too."""
    s = _product("noise", K, "dpmsolver++", thr)
    x = seeded(SHAPE, 3).cuda()
    nfe = 6
    s.sample(x, steps=nfe, order=2)
    torch.cuda.synchronize()
    n0 = cuda_backend.launch_count()
    s.sample(x, steps=nfe, order=2)
    torch.cuda.synchronize()
    n = cuda_backend.launch_count() - n0
    if not thr:
        assert n == 1 + nfe           # the first network input (dpm_replicate) + one fused launch per evaluation
    else:
        # the quantile of the one-condition thresholded run is the same launch sequence
        one = _one_condition_thresholded(nfe, x)
        assert n == 1 + 2 * nfe + (one - 1 - nfe), (n, one)


def _one_condition_thresholded(nfe, x):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    _, _, pns = schedules("sd")
    fn = new.model_wrapper(inner_net(), pns, guidance_type="classifier-free", condition=torch.ones(B, 1).cuda(),
                           unconditional_condition=torch.zeros(B, 1).cuda(), guidance_scale=7.5)
    s = new.DPM_Solver(fn, pns, correcting_x0_fn="dynamic_thresholding")
    s.sample(x, steps=nfe, order=2)
    torch.cuda.synchronize()
    n0 = ops.backend().launch_count()
    s.sample(x, steps=nfe, order=2)
    torch.cuda.synchronize()
    return ops.backend().launch_count() - n0
