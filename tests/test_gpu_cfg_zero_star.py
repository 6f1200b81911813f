"""CFG-Zero* on the H100: dpm_cfgzero_scale bit for bit against the executor's exact summation order and independent
of batch position; dpm_step_cfgzero bit for bit against the numpy executor on every form, parameterisation, dtype
pair, layout, tuning, dev_coef and at IEEE edges; sample() and UniPC.sample() against the executor and the
unmodified reference; graph replay with zero-init; launch counts; one launch beyond 2^31 elements."""
import dataclasses

import numpy as np
import pytest
import torch

from cfgzero_oracle import CFGZeroOracle, guided_net
from oracle import ref_loader
from test_cfg_zero_star import product_schedule, reference_schedule
from test_gpu_cfg_rescale import ulp_dist

pytestmark = pytest.mark.gpu
DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16"), ("bf16", "f32"), ("f16", "f32")]   # (model, state)
COEF = dict(a=0.9, c0=-0.3, c1=0.2, c2=0.1, w0=1.5, w1=0.7, w2=0.4, w3=0.6, w4=0.3)
W = 4.5


def unaligned(t):
    """A contiguous copy of t whose storage starts one element past an aligned address."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def cpu(a):
    t = {f.name: getattr(a, f.name).cpu() for f in dataclasses.fields(a) if torch.is_tensor(getattr(a, f.name))}
    t["coef_dev"] = None
    return dataclasses.replace(a, **t)


def same(got, want):
    """Bit for bit, NaN matching NaN."""
    g, w = got.float().cpu().numpy(), want.float().cpu().numpy()
    assert g.shape == w.shape
    assert np.array_equal(np.isnan(g), np.isnan(w)), "NaN pattern differs"
    m = ~np.isnan(g)
    assert g[m].tobytes() == w[m].tobytes(), float(np.abs(g[m].astype(np.float64) - w[m]).max())


def _args(param, px0, md, sd, Bn, ps, gen, form=0, layout="c", per_sample=False, dev_coef=False):
    from dpm_solver_b200.ops import StepArgs
    shape = (Bn, 4, ps // 16, 4) if layout == "cl" else (Bn, ps)

    def t(dtype, scale=1.0, shift=0.0):
        v = (torch.randn(shape, generator=gen) * scale + shift).to(dtype).cuda()
        return v.contiguous(memory_format=torch.channels_last) if layout == "cl" else v
    x = t(sd)
    al, sg = (0.8, 0.6) if param != 5 else (0.2, 0.45)
    ec = t(md, 1.3, 0.2)
    eu = (0.6 * ec.float() + t(torch.float32, 0.5)).to(md)
    a = StepArgs(form=form, n_model=2, x=x if form else None, xe=x, e_cond=ec, e_uncond=eu,
                 param=param, predict_x0=px0, guidance=W, alpha_e=al, sigma_e=sg, state_dtype=sd, want_m_out=True,
                 per_sample=ps, m1=t(sd) if form in (2, 3, 4, 5, 6) else None,
                 m2=t(sd) if form in (3, 5, 6) else None, **COEF)
    a.c0_on_old = form == 4 and param % 2 == 1
    if per_sample:
        a.guidance_b = torch.tensor([1.0, W, -2.0, 0.5, 3.0][:Bn] + [W] * max(0, Bn - 5), dtype=torch.float32).cuda()
    if dev_coef:
        v = [COEF[k] for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4")] + [al, sg]
        a.coef_dev = torch.tensor(v + [0.] * 5, dtype=torch.float32).cuda()
    return a


# ---- the s* pass -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("ps", [8, 104, 8192 + 16, 3 * 64 * 64, 7, 9, 8193])
def test_s_star_bit_exact(cuda_backend, dt, ps):
    gen = torch.Generator().manual_seed(ps)
    o = CFGZeroOracle()
    for layout in ("c", "cl") if ps % 64 == 0 else ("c",):
        a = _args(0, True, DT[dt], DT[dt], 3, ps, gen, layout=layout)
        s = cuda_backend.cfgzero_scale(a.e_cond, a.e_uncond)
        assert torch.equal(s, cuda_backend.cfgzero_scale(a.e_cond, a.e_uncond)), "s* is not deterministic"
        same(s, o.cfgzero_scale(a.e_cond.cpu(), a.e_uncond.cpu()))
        for b in range(3):      # a sample alone, in fresh (differently aligned) storage, gives the same bits
            sb = cuda_backend.cfgzero_scale(a.e_cond[b:b + 1].clone(), a.e_uncond[b:b + 1].clone())
            assert torch.equal(sb[0], s[b])
    # unaligned storage takes the element-wise path: the same bits
    a = _args(0, True, DT[dt], DT[dt], 2, ps, gen)
    ec, eu = unaligned(a.e_cond), unaligned(a.e_uncond)
    same(cuda_backend.cfgzero_scale(ec, eu), o.cfgzero_scale(ec.cpu(), eu.cpu()))
    same(cuda_backend.cfgzero_scale(ec, eu), cuda_backend.cfgzero_scale(a.e_cond, a.e_uncond))


def test_s_star_ieee_edges(cuda_backend):
    c = torch.randn(4, 1000).cuda()
    u = torch.randn(4, 1000).cuda()
    u[0] = 0.0                          # s* = 0/(0 + 1e-8) = 0
    u[1, 17] = float("inf")             # inf*c and inf/inf: NaN
    c[2, 3] = float("nan")
    s = cuda_backend.cfgzero_scale(c, u).cpu()
    assert s[0] == 0.0 and torch.isnan(s[1]) and torch.isnan(s[2]) and torch.isfinite(s[3])
    same(s, CFGZeroOracle().cfgzero_scale(c.cpu(), u.cpu()))


# ---- the step ----------------------------------------------------------------------------------------------------------

def _check_step(be, a):
    a.cfgzero_s = be.cfgzero_scale(a.e_cond, a.e_uncond)
    m, o = be.step(a)
    mw, ow = CFGZeroOracle().step(cpu(a))
    same(m, mw)
    if ow is not None:
        same(o, ow)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])      # whole packets per sample / tails and the generic kernel
def test_step_vs_executor(cuda_backend, pair, ps):
    gen = torch.Generator().manual_seed(ps)
    for form in range(7):
        for param in range(6):
            for px0 in (False, True):
                _check_step(cuda_backend, _args(param, px0, DT[pair[0]], DT[pair[1]], 5, ps, gen, form,
                                                per_sample=(form + param) % 2 == 1))


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
def test_step_layouts_tunings_and_dev_coef(cuda_backend, pair):
    gen = torch.Generator().manual_seed(7)
    for form in (0, 1, 5):
        _check_step(cuda_backend, _args(4, True, DT[pair[0]], DT[pair[1]], 4, 16 * 12, gen, form, "cl"))
        if form:
            for param in range(5):
                _check_step(cuda_backend, _args(param, param % 2 == 0, DT[pair[0]], DT[pair[1]], 4, 3 * 40, gen, form,
                                                per_sample=param == 1, dev_coef=True))
    # an unaligned view of the halves: the generic kernel
    a = _args(0, True, DT[pair[0]], DT[pair[1]], 2, 8 * 33, gen, 1)
    a.e_cond = unaligned(a.e_cond)
    _check_step(cuda_backend, a)
    try:
        for variant, threads, ctas in ((2, 0, 0), (0, 64, 1), (0, 128, 2), (2, 512, 4), (1, 256, 0)):
            cuda_backend.set_tuning(variant, threads, ctas)
            _check_step(cuda_backend, _args(0, True, DT[pair[0]], DT[pair[1]], 3, 8 * 1024 * 6, gen, 5,
                                            per_sample=threads == 128))
    finally:
        cuda_backend.set_tuning(2, 0, 0)


@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])
def test_step_ieee_edges(cuda_backend, ps):
    """u = 0 (s* = 0, g = w*c), an infinite and a NaN half in one sample each: the rows match the executor bit for bit,
    the non-finite ones propagate and the others stay finite."""
    gen = torch.Generator().manual_seed(3)
    for param in (0, 4):
        a = _args(param, True, torch.float32, torch.float32, 4, ps, gen, 1, per_sample=True)
        a.e_uncond[1] = 0.0             # (row 0 has scale 1: the bypass)
        a.e_uncond[2, 5] = float("inf")
        a.e_cond[3, 7] = float("nan")
        _check_step(cuda_backend, a)
        s = a.cfgzero_s.cpu()
        assert s[1] == 0.0 and torch.isnan(s[2]) and torch.isnan(s[3]) and torch.isfinite(s[0])


# ---- end to end --------------------------------------------------------------------------------------------------------

def net(x, t, c):
    """Products and sums only: the same bits on the CPU and on the GPU for fp32 inputs."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.45 * x + 0.05 * cc * x - 0.1 + 0.05 * cc


def wrap(mt, ns, device, w=W, model=net, B=2, **kw):
    import dpm_solver_b200 as new
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free",
                             condition=torch.ones(B, 1, device=device), unconditional_condition=torch.zeros(B, 1, device=device),
                             guidance_scale=w, cfg_zero_star=True, **kw)


def _on(be):
    from dpm_solver_b200 import ops
    old = ops._backend
    ops.set_backend(be)
    return old


def _runs(be, mt, device, solver, sd=None, shape=(2, 4, 16, 16), **kw):
    """(first call, second call, fresh solver) of one configuration."""
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    old = _on(be)
    try:
        ns = product_schedule(mt)
        fn = wrap(mt, ns, device, B=shape[0], cfg_zero_init_steps=1)
        x = torch.randn(shape, generator=torch.Generator().manual_seed(0)).to(device)
        mk = (lambda: new.UniPC(fn, ns, state_dtype=sd, **kw)) if solver == "unipc" else \
            (lambda: new.DPM_Solver(fn, ns, state_dtype=sd, **kw))
        skw = dict(steps=6, order=2) if solver == "unipc" else dict(steps=6, order=3, method="singlestep")
        s = mk()
        return [s.sample(x.clone(), **skw), s.sample(x.clone(), **skw), mk().sample(x.clone(), **skw)]
    finally:
        ops.set_backend(old)


@pytest.mark.parametrize("mt", ["noise", "v", "flow", "edm"])
@pytest.mark.parametrize("solver", ["dpm", "unipc"])
def test_sample_vs_executor(cuda_backend, mt, solver):
    ys = _runs(cuda_backend, mt, "cuda", solver)
    yw = _runs(CFGZeroOracle(), mt, "cpu", solver)[0]
    for y in ys:
        same(y, yw)
    # bf16 state: the network itself then computes in bf16, where torch's CPU and CUDA kernels round a python scalar
    # differently; the three device runs are bit-identical and the executor's run is within bf16 rounding
    ys = _runs(cuda_backend, mt, "cuda", solver, torch.bfloat16)
    yw = _runs(CFGZeroOracle(), mt, "cpu", solver, torch.bfloat16)[0].float()
    assert torch.equal(ys[0], ys[1]) and torch.equal(ys[0], ys[2])
    err = float((ys[0].float().cpu() - yw).abs().max() / yw.abs().max())
    assert err <= 2e-2, err
    yt = _runs(cuda_backend, mt, "cuda", "dpm", correcting_x0_fn="dynamic_thresholding")
    ytw = _runs(CFGZeroOracle(), mt, "cpu", "dpm", correcting_x0_fn="dynamic_thresholding")[0]
    for y in yt:
        same(y, ytw)


@pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")
@pytest.mark.parametrize("mt", ["noise", "x_start", "v", "score", "flow", "edm"])
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
def test_fp32_sample_vs_reference(cuda_backend, mt, algo):
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    shape, K = (4, 4, 64, 64), 1
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1))
    ns = product_schedule(mt)
    y = new.DPM_Solver(wrap(mt, ns, "cuda", B=4, cfg_zero_init_steps=K), ns, algorithm_type=algo).sample(
        x.cuda(), steps=6, order=2).cpu()
    rns = reference_schedule(mt)
    g = guided_net(net, torch.zeros(4, 1), torch.ones(4, 1), W, K)
    if mt in ("flow", "edm"):
        from flow_oracle import reference_solver as flow_solver
        from edm_oracle import reference_solver as edm_solver
        rs = (flow_solver if mt == "flow" else edm_solver)(g, rns, algo)
    else:
        rs = ref.DPM_Solver(ref.model_wrapper(g, rns, model_type=mt), rns, algorithm_type=algo)
    same(y, rs.sample(x, steps=6, order=2, method="multistep"))


@pytest.mark.parametrize("mt", ["noise", "flow"])
def test_capture_with_zero_init_replays_bit_identically(cuda_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    s = new.DPM_Solver(wrap(mt, ns, "cuda", cfg_zero_init_steps=2), ns)
    x = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(2)).cuda()
    skw = dict(steps=6, order=2)
    eager = s.sample(x.clone(), **skw)
    g = s.capture(x, **skw)
    y1 = g(x).clone()
    y2 = g(x).clone()
    assert torch.equal(y1, y2) and torch.equal(y1, eager)


@pytest.mark.parametrize("thr", [False, True])
def test_launch_counts(cuda_backend, thr):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    counts, calls = {}, {}
    for cfz, K in ((False, 0), (True, 0), (True, 2)):
        n = []

        def counted(x, t, c, n=n):
            n.append(1)
            return net(x, t, c)
        kw = dict(cfg_zero_star=True, cfg_zero_init_steps=K) if cfz else {}
        fn = new.model_wrapper(counted, ns, guidance_type="classifier-free", condition=torch.ones(2, 1).cuda(),
                               unconditional_condition=torch.zeros(2, 1).cuda(), guidance_scale=W, **kw)
        s = new.DPM_Solver(fn, ns, correcting_x0_fn="dynamic_thresholding" if thr else None)
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)    # plans, tables and prepared launches cached
        torch.cuda.synchronize()
        before = cuda_backend.launch_count()
        n.clear()
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)
        counts[(cfz, K)], calls[(cfz, K)] = cuda_backend.launch_count() - before, len(n)
    per = 3 if thr else 2
    # 6 evaluations: +2 s* launches each, +1 materialising launch each under thresholding
    assert counts[(True, 0)] - counts[(False, 0)] == 6 * per, counts
    # a zero-init evaluation: no network call, no s* pass, one step launch (+ the quantile under thresholding)
    # (and the run's first network input is no longer a dpm_duplicate launch: the zero-init step writes it)
    assert calls[(True, 2)] == calls[(True, 0)] - 2
    assert counts[(True, 0)] - counts[(True, 2)] == 2 * per + 1, counts


def test_per_sample_rows_equal_scalar_runs(cuda_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    scales = [W, 1.0, 2.5, -1.0]
    x = torch.randn((4, 4, 128, 128), generator=torch.Generator().manual_seed(9)).cuda()
    y = new.DPM_Solver(wrap("flow", ns, "cuda", w=torch.tensor(scales).cuda(), B=4, cfg_zero_init_steps=1), ns,
                       state_dtype=torch.bfloat16).sample(x, steps=6, order=2)
    for b, s in enumerate(scales):
        fb = wrap("flow", ns, "cuda", w=s, B=1, cfg_zero_init_steps=1)
        yb = new.DPM_Solver(fb, ns, state_dtype=torch.bfloat16).sample(x[b:b + 1].clone(), steps=6, order=2)
        assert torch.equal(y[b:b + 1], yb), b


def test_launch_beyond_2_31_elements(cuda_backend):
    """One s* pass and one step over 2^31 + 1003 elements (bf16, one sample: the element-wise paths) against separate
    torch CUDA ops: s* within an ulp of torch's fp64 sums, the step bit for bit from the device's s*."""
    from dpm_solver_b200.ops import StepArgs
    n = 2 ** 31 + 1003
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((1, n), generator=g, device="cuda", dtype=torch.bfloat16)
    ec = torch.randn((1, n), generator=g, device="cuda", dtype=torch.bfloat16)
    eu = torch.randn((1, n), generator=g, device="cuda", dtype=torch.bfloat16)
    s = cuda_backend.cfgzero_scale(ec, eu)
    cu = uu = 0.0
    for k in range(0, n, 2 ** 28):
        c64, u64 = ec[:, k:k + 2 ** 28].double(), eu[:, k:k + 2 ** 28].double()
        cu += float((c64 * u64).sum())
        uu += float((u64 * u64).sum())
        del c64, u64
    assert ulp_dist(s.cpu().numpy(), np.array([cu / (uu + 1e-8)], np.float32)) <= 1
    a = StepArgs(form=1, n_model=2, x=x, xe=x, e_cond=ec, e_uncond=eu, param=4, predict_x0=True, guidance=W,
                 alpha_e=0.8, sigma_e=0.6, a=0.9, c0=-0.3, state_dtype=torch.bfloat16, per_sample=n, cfgzero_s=s)
    _, out = cuda_backend.step(a)
    sv = s.reshape(1, 1)
    for k in range(0, n, 2 ** 28):
        sl = slice(k, k + 2 ** 28)
        us = eu[:, sl].float() * sv
        gg = us + W * (ec[:, sl].float() - us)
        x0 = (x[:, sl].float() - 0.6 * gg).to(torch.bfloat16).float()     # the buffered value, in the state dtype
        want = (0.9 * x[:, sl].float() + (-0.3) * x0).to(torch.bfloat16)
        assert torch.equal(out[:, sl], want), k
