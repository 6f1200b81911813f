"""CFG++ on the H100: dpm_step_cfgpp bit for bit against the numpy executor (tests/cfgpp_oracle.py) on both forms, every
parameterisation and dtype pair, scalar and per-sample scales, with and without out2 / m_out, tails, unaligned views,
channels_last, every tuning and IEEE edge operands; one launch beyond 2^31 elements against separate torch ops; seeded
sample() runs against the executor (repeated calls, a fresh solver, capture() replay, intermediates, bf16 state); and a
condition-blind network on the device equal to the unmodified reference and to the plain run."""
import dataclasses

import numpy as np
import pytest
import torch

from cfgpp_oracle import CFGPPOracle
from oracle import ref_loader
from step_edges import DIV_OK, DIV_REFUSED, edge_pool
from test_cfg_pp import blind, product_schedule, reference_solver

pytestmark = pytest.mark.gpu
DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16"), ("bf16", "f32"), ("f16", "f32")]   # (model, state)
COEF = dict(a=0.9, c0=0.3, c1=-0.2, w0=1.5)
G_W = 0.8          # the alpha_t word g
LAM = 0.6


def unaligned(t):
    """A contiguous copy of t whose storage starts one element past an aligned address."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def cpu(a):
    t = {f.name: getattr(a, f.name).cpu() for f in dataclasses.fields(a) if torch.is_tensor(getattr(a, f.name))}
    return dataclasses.replace(a, **t)


def same(got, want):
    """Bit for bit, NaN matching NaN."""
    g, w = got.float().cpu().numpy(), want.float().cpu().numpy()
    assert g.shape == w.shape
    assert np.array_equal(np.isnan(g), np.isnan(w)), "NaN pattern differs"
    m = ~np.isnan(g)
    assert g[m].tobytes() == w[m].tobytes(), float(np.abs(g[m].astype(np.float64) - w[m]).max())


def _args(param, md, sd, Bn, ps, gen, form=1, layout="c", per_sample=False, out2=False, m_out=True):
    from dpm_solver_b200.ops import StepArgs
    shape = (Bn, 4, ps // 16, 4) if layout == "cl" else (Bn, ps)

    def t(dtype, scale=1.0, shift=0.0):
        v = (torch.randn(shape, generator=gen) * scale + shift).to(dtype).cuda()
        return v.contiguous(memory_format=torch.channels_last) if layout == "cl" else v
    x = t(sd)
    al, sg = (0.8, 0.6) if param != 5 else (0.2, 0.45)
    ec = t(md, 1.3, 0.2)
    eu = (0.6 * ec.float() + t(torch.float32, 0.5)).to(md)
    a = StepArgs(form=form, n_model=2, x=x, xe=x, e_cond=ec, e_uncond=eu, param=param, predict_x0=True,
                 guidance=LAM, alpha_e=al, sigma_e=sg, state_dtype=sd, want_m_out=m_out, per_sample=ps,
                 m1=t(sd) if form == 4 else None, cfgpp_g=G_W, **COEF)
    if per_sample:
        a.guidance_b = torch.tensor([1.0, LAM, -2.0, 0.25, 3.0][:Bn] + [LAM] * max(0, Bn - 5),
                                    dtype=torch.float32).cuda()
    if out2:
        x_in = torch.empty((2 * Bn,) + tuple(shape[1:]), dtype=sd, device="cuda")
        if layout == "cl":
            x_in = x_in.contiguous(memory_format=torch.channels_last)
        a.out, a.out2 = x_in[:Bn], x_in[Bn:]
    return a


def _check(be, a):
    m, o = be.step(a)
    mw, ow = CFGPPOracle().step(cpu(a))
    if a.want_m_out:
        same(m, mw)
    else:
        assert m is None
    same(o, ow)
    if a.out2 is not None:
        same(a.out2, ow)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])      # whole packets per sample / tails and the generic kernel
def test_step_vs_executor(cuda_backend, pair, ps):
    gen = torch.Generator().manual_seed(ps)
    k = 0
    for form in (1, 4):
        for param in range(6):
            for per_sample in (False, True):
                k += 1
                _check(cuda_backend, _args(param, DT[pair[0]], DT[pair[1]], 5, ps, gen, form, per_sample=per_sample,
                                           out2=k % 2 == 0, m_out=k % 3 != 0))


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
def test_step_layouts_and_tunings(cuda_backend, pair):
    gen = torch.Generator().manual_seed(7)
    md, sd = DT[pair[0]], DT[pair[1]]
    for form in (1, 4):
        for param in (0, 2, 4):
            _check(cuda_backend, _args(param, md, sd, 4, 16 * 12, gen, form, "cl", per_sample=param == 2, out2=True))
    # unaligned views: the generic kernel
    for form in (1, 4):
        a = _args(0, md, sd, 2, 8 * 33, gen, form, per_sample=form == 4)
        a.e_cond = unaligned(a.e_cond)
        _check(cuda_backend, a)
        a = _args(4, md, sd, 2, 8 * 33, gen, form)
        a.x = a.xe = unaligned(a.x)
        _check(cuda_backend, a)
    # a state the network was not evaluated at (xe != x): both read
    a = _args(1, md, sd, 3, 16 * 64, gen, 4)
    a.xe = a.x + 0.25
    _check(cuda_backend, a)
    try:
        for variant, threads, ctas in ((2, 0, 0), (0, 64, 1), (0, 128, 2), (2, 512, 4), (1, 256, 0), (0, 32, 32)):
            cuda_backend.set_tuning(variant, threads, ctas)
            for form in (1, 4):
                _check(cuda_backend, _args(form % 3, md, sd, 3, 8 * 1024 * 6 + 8, gen, form,
                                           per_sample=threads == 128, out2=True))
    finally:
        cuda_backend.set_tuning(2, 0, 0)


@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])
@pytest.mark.parametrize("param", [0, 1, 2, 4, 5])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
def test_step_ieee_edges(cuda_backend, ps, param, pair):
    """tests/step_edges.py's values scattered over both halves, x and m1, and divisors on both sides of the constant
    division's acceptance test: the executor's bits, NaN for NaN."""
    gen = torch.Generator().manual_seed(11)
    md, sd = DT[pair[0]], DT[pair[1]]
    for form in (1, 4):
        a = _args(param, md, sd, 4, ps, gen, form, per_sample=True)
        n = a.x.numel()
        for name, t in (("x", a.x), ("e_cond", a.e_cond), ("e_uncond", a.e_uncond), ("m1", a.m1)):
            if t is None:
                continue
            edges = torch.from_numpy(edge_pool(t.dtype))
            idx = torch.randperm(n, generator=gen)[:edges.numel()]
            t.view(-1)[idx.cuda()] = edges.to(t.dtype).cuda()
        _check(cuda_backend, a)
        # alpha_e on both sides of the reciprocal-refinement division's acceptance test
        for al in [float(v) for v in DIV_OK + DIV_REFUSED]:
            _check(cuda_backend, dataclasses.replace(a, alpha_e=al))


def test_c_abi_refusals(cuda_backend):
    from dpm_solver_b200 import _lib
    gen = torch.Generator().manual_seed(1)
    a = _args(0, torch.float32, torch.float32, 2, 64, gen, 4)
    for bad in (dict(form=0), dict(form=5), dict(c0_on_old=True), dict(predict_x0=False),
                dict(thr=torch.ones(2).cuda()), dict(raw_round=1), dict(coef_dev=torch.zeros(16).cuda())):
        with pytest.raises((ValueError, RuntimeError)):
            cuda_backend.step(dataclasses.replace(a, **bad))
    assert _lib.lib().dpm_version() == 108


def test_launch_beyond_2_31_elements(cuda_backend):
    """One DIFF2 launch over 2^31 + 1003 bf16 elements (one sample; noise parameterisation) against separate torch CUDA
    ops in fp32, chunk by chunk: U, G, and the update."""
    from dpm_solver_b200.ops import StepArgs
    n = 2 ** 31 + 1003
    g = torch.Generator(device="cuda").manual_seed(0)
    bf = torch.bfloat16
    x = torch.randn((1, n), generator=g, device="cuda", dtype=bf)
    ec = torch.randn((1, n), generator=g, device="cuda", dtype=bf)
    eu = torch.randn((1, n), generator=g, device="cuda", dtype=bf)
    m1 = torch.randn((1, n), generator=g, device="cuda", dtype=bf)
    al, sg = 0.8, 0.6
    a = StepArgs(form=4, n_model=2, x=x, xe=x, e_cond=ec, e_uncond=eu, m1=m1, param=0, predict_x0=True, guidance=LAM,
                 alpha_e=al, sigma_e=sg, state_dtype=bf, want_m_out=True, cfgpp_g=G_W, **COEF)
    m, out = cuda_backend.step(a)
    f = lambda v: torch.tensor(v, dtype=torch.float32).item()
    # (a 0-dim CUDA divisor: torch divides by a host scalar through its reciprocal, which is not IEEE division)
    al_t = torch.tensor(al, dtype=torch.float32, device="cuda")
    for k in range(0, n, 2 ** 28):
        sl = slice(k, k + 2 ** 28)
        xf, c, u = x[:, sl].float(), ec[:, sl].float(), eu[:, sl].float()
        U = ((xf - f(sg) * u) / al_t).to(bf).float()
        G = ((xf - f(sg) * (u + f(LAM) * (c - u))) / al_t).to(bf).float()
        o = (f(COEF["a"]) * xf + f(COEF["c0"]) * U) + f(G_W) * (G - U)
        o = o + f(COEF["c1"]) * (f(COEF["w0"]) * (G - m1[:, sl].float()))
        assert torch.equal(m[:, sl], U.to(bf)), k
        assert torch.equal(out[:, sl], o.to(bf)), k
        del xf, c, u, U, G, o


# ---- end to end --------------------------------------------------------------------------------------------------------

def net(x, t, c):
    """Products and sums only: the same bits on the CPU and on the GPU for fp32 inputs."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.45 * x + 0.05 * cc * x - 0.1 + 0.05 * cc


def wrap(mt, ns, device, w=LAM, model=net, B=2, **kw):
    import dpm_solver_b200 as new
    if torch.is_tensor(w):
        w = w.to(device)
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free",
                             condition=torch.ones(B, 1, device=device),
                             unconditional_condition=torch.zeros(B, 1, device=device), guidance_scale=w, **kw)


def _runs(be, mt, device, sd=None, order=2, w=LAM, shape=(2, 4, 16, 16), **kw):
    """(first call, second call, fresh solver, the intermediates of a fourth) of one configuration."""
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    old = ops._backend
    ops.set_backend(be)
    try:
        ns = product_schedule(mt)
        fn = wrap(mt, ns, device, w=w, B=shape[0], cfg_pp=True)
        x = torch.randn(shape, generator=torch.Generator().manual_seed(0)).to(device)
        mk = lambda: new.DPM_Solver(fn, ns, state_dtype=sd)
        skw = dict(steps=7, order=order, **kw)
        s = mk()
        y1, y2 = s.sample(x.clone(), **skw), s.sample(x.clone(), **skw)
        y3 = mk().sample(x.clone(), **skw)
        _, inter = mk().sample(x.clone(), return_intermediate=True, **skw)
        return [y1, y2, y3] + list(inter)
    finally:
        ops.set_backend(old)


@pytest.mark.parametrize("mt", ["noise", "x_start", "v", "score", "flow", "edm"])
@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("w", ["scalar", "per_sample"])
def test_sample_vs_executor(cuda_backend, mt, order, w):
    ws = LAM if w == "scalar" else torch.tensor([1.0, 0.3])
    ys = _runs(cuda_backend, mt, "cuda", order=order, w=ws)
    yw = _runs(CFGPPOracle(), mt, "cpu", order=order, w=ws)
    for y in ys[:3]:
        same(y, yw[0])
    for y, z in zip(ys[3:], yw[3:]):
        same(y, z)
    if mt in ("noise", "flow"):
        # bf16 state: the network then computes in bf16, where torch's CPU and CUDA kernels round a python scalar
        # differently; the device runs are bit-identical to each other and the executor's within bf16 rounding
        ys = _runs(cuda_backend, mt, "cuda", torch.bfloat16, order=order, w=ws)
        yw = _runs(CFGPPOracle(), mt, "cpu", torch.bfloat16, order=order, w=ws)[0].float()
        assert torch.equal(ys[0], ys[1]) and torch.equal(ys[0], ys[2])
        err = float((ys[0].float().cpu() - yw).abs().max() / yw.abs().max())
        assert err <= 2e-2, err


@pytest.mark.parametrize("mt", ["noise", "flow"])
@pytest.mark.parametrize("w", ["scalar", "per_sample"])
def test_capture_replays_bit_identically(cuda_backend, mt, w):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    ws = LAM if w == "scalar" else torch.tensor([0.5, 0.3])
    s = new.DPM_Solver(wrap(mt, ns, "cuda", w=ws, cfg_pp=True), ns)
    x = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(2)).cuda()
    skw = dict(steps=6, order=2)
    eager = s.sample(x.clone(), **skw)
    g = s.capture(x, **skw)
    y1 = g(x).clone()
    y2 = g(x).clone()
    assert torch.equal(y1, y2) and torch.equal(y1, eager)


def test_launch_counts(cuda_backend):
    """One launch per evaluation, as the plain CFG run: the first network input from dpm_duplicate, then the update
    writes both halves of the next one."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    counts = {}
    for pp in (False, True):
        s = new.DPM_Solver(wrap("noise", ns, "cuda", w=0.5, cfg_pp=pp), ns)
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)
        torch.cuda.synchronize()
        before = cuda_backend.launch_count()
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)
        counts[pp] = cuda_backend.launch_count() - before
    assert counts[True] == counts[False] == 7, counts


@pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")
@pytest.mark.parametrize("mt", ["noise", "x_start", "v", "score", "flow", "edm"])
@pytest.mark.parametrize("order", [1, 2])
def test_condition_blind_fp32_equals_reference(cuda_backend, mt, order):
    import dpm_solver_b200 as new
    shape = (4, 4, 64, 64)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1))
    ns = product_schedule(mt)
    y = new.DPM_Solver(wrap(mt, ns, "cuda", w=torch.tensor([0.3, 1.0, 7.5, 0.6]), model=blind, B=4, cfg_pp=True),
                       ns).sample(x.cuda(), steps=6, order=order).cpu()
    yr = reference_solver(mt, lambda xx, tt: blind(xx, tt)).sample(x, steps=6, order=order, method="multistep")
    assert torch.equal(y, yr), float((y - yr).abs().max())


@pytest.mark.parametrize("mt", ["noise", "flow", "edm"])
@pytest.mark.parametrize("w", [0.3, 7.5])
def test_condition_blind_bf16_equals_plain_run(cuda_backend, mt, w):
    import dpm_solver_b200 as new
    shape = (4, 4, 64, 64)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(3)).cuda()
    ns = product_schedule(mt)
    kw = dict(steps=8, order=2)
    y = new.DPM_Solver(wrap(mt, ns, "cuda", w=w, model=blind, B=4, cfg_pp=True), ns,
                       state_dtype=torch.bfloat16).sample(x, **kw)
    y0 = new.DPM_Solver(wrap(mt, ns, "cuda", w=w, model=blind, B=4), ns, state_dtype=torch.bfloat16).sample(x, **kw)
    assert torch.equal(y, y0)
