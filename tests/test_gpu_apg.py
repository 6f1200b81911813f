"""Adaptive projected guidance on the H100: the words pass against fp64 words, dpm_step_apg against the numpy executor
bit for bit on every dispatch path and tuning, sample() and UniPC.sample() against the executor, graph replay with
momentum, launch counts, per-sample rows against their scalar runs and one launch beyond 2^31 elements."""
import dataclasses

import numpy as np
import pytest
import torch

from apg_oracle import APGOracle
from test_apg import W, product_schedule, rel_err, wrap
from test_gpu_cfg_rescale import ulp_dist

pytestmark = pytest.mark.gpu
DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16"), ("bf16", "f32"), ("f16", "f32")]   # (model, state)
COEF = dict(a=0.9, c0=-0.3, c1=0.2, c2=0.1, w0=1.5, w1=0.7, w2=0.4, w3=0.6, w4=0.3)


def cpu(a):
    t = {f.name: getattr(a, f.name).cpu() for f in dataclasses.fields(a) if torch.is_tensor(getattr(a, f.name))}
    t["coef_dev"] = None
    return dataclasses.replace(a, **t)


def _args(param, px0, md, sd, Bn, ps, gen, form=0, layout="c", per_sample=False, dev_coef=False):
    from dpm_solver_b200.ops import StepArgs
    shape = (Bn, 4, ps // 16, 4) if layout == "cl" else (Bn, ps)

    def t(dtype, scale=1.0, shift=0.0):
        v = (torch.randn(shape, generator=gen) * scale + shift).to(dtype).cuda()
        return v.contiguous(memory_format=torch.channels_last) if layout == "cl" else v
    x = t(sd)
    al, sg = (0.8, 0.6) if param != 5 else (0.2, 0.45)
    a = StepArgs(form=form, n_model=2, x=x if form else None, xe=x, e_cond=t(md, 1.3, 0.2), e_uncond=t(md),
                 param=param, predict_x0=px0, guidance=W, alpha_e=al, sigma_e=sg, alpha_t=0.8, sigma_t=0.6,
                 state_dtype=sd, want_m_out=True, per_sample=ps,
                 m1=t(sd) if form in (2, 3, 4, 5, 6) else None, m2=t(sd) if form in (3, 5, 6) else None, **COEF)
    a.c0_on_old = form == 4 and param % 2 == 1
    if per_sample:
        a.guidance_b = torch.tensor([1.0, W, -2.0, 0.5, 3.0][:Bn] + [W] * max(0, Bn - 5), dtype=torch.float32).cuda()
    if dev_coef:
        v = [COEF[k] for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4")] + [0.8, 0.6]
        a.coef_dev = torch.tensor(v + [0.] * 5, dtype=torch.float32).cuda()
        a.alpha_e, a.sigma_e = 0.8, 0.6
    return a


# ---- the words pass ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("ps", [8, 104, 8192 + 16, 3 * 64 * 64, 7, 9, 8193])
def test_words_vs_fp64(cuda_backend, dt, ps):
    gen = torch.Generator().manual_seed(ps)
    o = APGOracle()
    for param in range(6):
        for eta, r, beta in ((0.0, 0.0, 0.0), (0.5, 1.0, -0.5), (1.0, 1e6, 0.3)):
            a = _args(param, True, DT[dt], DT["f32"] if dt == "f32" else DT[dt], 3, ps, gen, per_sample=param == 2)
            r_prev = torch.randn(a.e_cond.shape, generator=gen).cuda() if beta else None
            r_out = torch.empty(a.e_cond.shape, device="cuda") if beta else None
            w = cuda_backend.apg_words(a, eta, r, beta, r_prev, r_out)
            w2 = cuda_backend.apg_words(a, eta, r, beta, r_prev, None)
            assert w.cpu().numpy().tobytes() == w2.cpu().numpy().tobytes(), "words are not deterministic"
            ro_cpu = torch.empty(a.e_cond.shape) if beta else None
            want = o.apg_words(cpu(a), eta, r, beta, None if r_prev is None else r_prev.cpu(), ro_cpu)
            assert ulp_dist(w.cpu().numpy(), want.numpy()) <= 1, (param, eta, r, beta)
            if beta:
                assert torch.equal(r_out.cpu(), ro_cpu)
            for b in range(3):      # a sample alone (fresh storage) gives the bits it has inside the batch
                ab = dataclasses.replace(a, xe=a.xe[b:b + 1].clone(), e_cond=a.e_cond[b:b + 1].clone(),
                                         e_uncond=a.e_uncond[b:b + 1].clone(),
                                         guidance_b=None if a.guidance_b is None else a.guidance_b[b:b + 1].clone())
                wb = cuda_backend.apg_words(ab, eta, r, beta, None if r_prev is None else r_prev[b:b + 1].clone(), None)
                assert torch.equal(wb.cpu()[:, 0], w.cpu()[:, b])


def test_words_channels_last_and_dev_coef(cuda_backend):
    gen = torch.Generator().manual_seed(5)
    o = APGOracle()
    for dc in (False, True):
        a = _args(0, True, DT["bf16"], DT["bf16"], 4, 16 * 24, gen, layout="c" if dc else "cl", dev_coef=dc)
        w = cuda_backend.apg_words(a, 0.3, 2.0, 0.0)
        assert ulp_dist(w.cpu().numpy(), o.apg_words(cpu(a), 0.3, 2.0, 0.0).numpy()) <= 1


# ---- the step ----------------------------------------------------------------------------------------------------------

def _check_step(be, a, beta=0.0):
    r_out = None
    if beta:
        r_out = torch.empty(a.xe.shape, device="cuda")
        if a.xe.dim() == 4 and not a.xe.is_contiguous():
            r_out = r_out.contiguous(memory_format=torch.channels_last)
    a.apg_words = be.apg_words(a, 0.2, 3.0, beta, None, r_out)
    a.apg_r = r_out
    m, o = be.step(a)
    mw, ow = APGOracle().step(cpu(a))
    assert m.float().cpu().numpy().tobytes() == mw.float().numpy().tobytes()
    if ow is not None:
        assert o.float().cpu().numpy().tobytes() == ow.float().numpy().tobytes()


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])      # whole packets per sample / tails and the generic kernel
def test_step_vs_executor(cuda_backend, pair, ps):
    gen = torch.Generator().manual_seed(ps)
    for form in range(7):
        for param in range(6):
            for px0 in (False, True):
                for beta in (0.0, -0.5):
                    _check_step(cuda_backend, _args(param, px0, DT[pair[0]], DT[pair[1]], 5, ps, gen, form,
                                                    per_sample=form % 2 == 1), beta)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
def test_step_layouts_tunings_and_dev_coef(cuda_backend, pair):
    gen = torch.Generator().manual_seed(7)
    for form in (0, 1, 5):
        _check_step(cuda_backend, _args(0, True, DT[pair[0]], DT[pair[1]], 4, 16 * 12, gen, form, "cl"), -0.5)
        if form:
            _check_step(cuda_backend, _args(2, False, DT[pair[0]], DT[pair[1]], 4, 3 * 40, gen, form, dev_coef=True))
    # every tuning: the grid-stride loop of the direct kernel over ~3 passes of the largest capped grid
    try:
        for threads, ctas in ((0, 0), (64, 1), (128, 2), (512, 4)):
            cuda_backend.set_tuning(2, threads, ctas)
            _check_step(cuda_backend, _args(0, True, DT[pair[0]], DT[pair[1]], 3, 8 * 1024 * 6, gen, 5), -0.5)
    finally:
        cuda_backend.set_tuning(2, 0, 0)


# ---- end to end --------------------------------------------------------------------------------------------------------

SHAPE = (2, 4, 16, 16)


def _x(seed=0):
    return torch.randn(SHAPE, generator=torch.Generator().manual_seed(seed))


def _on(be):
    from dpm_solver_b200 import ops
    old = ops._backend
    ops.set_backend(be)
    return old


def _run(be, mt, device, solver="dpm", sd=None, **kw):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    old = _on(be)
    try:
        ns = product_schedule(mt)
        fn = wrap(mt, ns, uc=torch.zeros(2, 1, device=device), c=torch.ones(2, 1, device=device),
                  apg_eta=0.1, apg_norm_threshold=20.0, apg_momentum=-0.5)
        if solver == "unipc":
            s = new.UniPC(fn, ns, state_dtype=sd)
            return s.sample(_x().to(device), steps=6, order=2)
        s = new.DPM_Solver(fn, ns, state_dtype=sd, **kw)
        return s.sample(_x().to(device), steps=6, order=3, method="singlestep")
    finally:
        ops.set_backend(old)


@pytest.mark.parametrize("mt", ["noise", "v", "flow", "edm"])
@pytest.mark.parametrize("solver", ["dpm", "unipc"])
def test_sample_vs_executor(cuda_backend, mt, solver):
    y = _run(cuda_backend, mt, "cuda", solver).cpu()
    yw = _run(APGOracle(), mt, "cpu", solver)
    # the words differ from the executor's fp64 sums by at most an ulp
    assert rel_err(y, yw) <= 1e-5
    y16 = _run(cuda_backend, mt, "cuda", solver, sd=torch.bfloat16).float().cpu()
    y16w = _run(APGOracle(), mt, "cpu", solver, sd=torch.bfloat16).float()
    assert rel_err(y16, y16w) <= 2e-2
    yt = _run(cuda_backend, mt, "cuda", "dpm", correcting_x0_fn="dynamic_thresholding").cpu()
    ytw = _run(APGOracle(), mt, "cpu", "dpm", correcting_x0_fn="dynamic_thresholding")
    assert rel_err(yt, ytw) <= 1e-5


def test_capture_replays_bit_identically(cuda_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    fn = wrap("noise", ns, uc=torch.zeros(2, 1).cuda(), c=torch.ones(2, 1).cuda(), apg_eta=0.0, apg_momentum=-0.5,
              apg_norm_threshold=5.0)
    s = new.DPM_Solver(fn, ns)
    x = _x(2).cuda()
    skw = dict(steps=6, order=2, method="multistep")
    eager = s.sample(x.clone(), **skw)
    g = s.capture(x, **skw)
    y1 = g(x).clone()
    y2 = g(x).clone()
    assert torch.equal(y1, y2) and torch.equal(y1, eager)


@pytest.mark.parametrize("thr", [False, True])
def test_launch_counts(cuda_backend, thr):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    counts = {}
    for apg in (None, 0.0):
        kw = {} if apg is None else dict(apg_eta=apg, apg_momentum=-0.5)
        fn = wrap("noise", ns, uc=torch.zeros(2, 1).cuda(), c=torch.ones(2, 1).cuda(), **kw)
        s = new.DPM_Solver(fn, ns, correcting_x0_fn="dynamic_thresholding" if thr else None)
        s.sample(_x().cuda(), steps=6, order=2)           # plans, tables and prepared launches cached
        torch.cuda.synchronize()
        before = cuda_backend.launch_count()
        s.sample(_x().cuda(), steps=6, order=2)
        counts[apg] = cuda_backend.launch_count() - before
    # 6 evaluations: +2 words launches each, +1 materialising launch each under thresholding
    assert counts[0.0] - counts[None] == 6 * (3 if thr else 2), counts


def test_per_sample_rows_equal_scalar_runs(cuda_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    scales = [W, 1.0, 2.5, -1.0]
    shape = (4, 4, 128, 128)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(9)).cuda()
    kw = dict(apg_eta=0.2, apg_norm_threshold=30.0, apg_momentum=-0.5)
    uc, c = torch.zeros(4, 1).cuda(), torch.ones(4, 1).cuda()
    fn = wrap("noise", ns, w=torch.tensor(scales).cuda(), uc=uc, c=c, **kw)
    y = new.DPM_Solver(fn, ns, state_dtype=torch.bfloat16).sample(x, steps=6, order=2)
    for b, s in enumerate(scales):
        fb = wrap("noise", ns, w=s, uc=uc[b:b + 1], c=c[b:b + 1], **kw)
        yb = new.DPM_Solver(fb, ns, state_dtype=torch.bfloat16).sample(x[b:b + 1].clone(), steps=6, order=2)
        assert torch.equal(y[b:b + 1], yb), b


def test_launch_beyond_2_31_elements(cuda_backend):
    """One words pass and one step over 2^31 + 2^13 elements (bf16), spot-checked per sample against the executor."""
    from dpm_solver_b200.ops import StepArgs
    ps = 2 ** 24
    Bn = 2 ** 31 // ps + 1
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((Bn, ps), generator=g, device="cuda", dtype=torch.bfloat16)
    ec = torch.randn((Bn, ps), generator=g, device="cuda", dtype=torch.bfloat16)
    eu = torch.randn((Bn, ps), generator=g, device="cuda", dtype=torch.bfloat16)
    a = StepArgs(form=1, n_model=2, x=x, xe=x, e_cond=ec, e_uncond=eu, param=0, predict_x0=True, guidance=W,
                 alpha_e=0.8, sigma_e=0.6, a=0.9, c0=-0.3, state_dtype=torch.bfloat16, per_sample=ps)
    a.apg_words = cuda_backend.apg_words(a, 0.3, 0.0, 0.0)
    _, out = cuda_backend.step(a)
    words = a.apg_words.cpu()
    for b in (0, Bn - 1):
        ab = dataclasses.replace(a, x=x[b:b + 1].cpu(), xe=x[b:b + 1].cpu(), e_cond=ec[b:b + 1].cpu(),
                                 e_uncond=eu[b:b + 1].cpu(), apg_words=words[:, b:b + 1].contiguous())
        assert ulp_dist(words[:, b].numpy(), APGOracle().apg_words(ab, 0.3, 0.0, 0.0)[:, 0].numpy()) <= 1
        _, ow = APGOracle().step(ab)
        assert torch.equal(out[b:b + 1].cpu(), ow)
