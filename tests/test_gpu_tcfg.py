"""TCFG on the H100: dpm_tcfg_words bit for bit against the executor's exact summation order, deterministic and
independent of batch position; dpm_step_tcfg bit for bit against the numpy executor on every form, parameterisation,
dtype pair, layout, tuning, dev_coef and at IEEE edges; sample(), UniPC and the device adaptive controller against the
executor; capture() replay; the condition-blind identity against the unmodified reference; one launch beyond 2^31
elements."""
import numpy as np
import pytest
import torch

from oracle import ref_loader
from step_edges import scatter_edges
from tcfg_oracle import TCFGOracle, guided_net, words_closed_form
from test_gpu_cfg_zero_star import DT, PAIRS, W, _args, _on, cpu, same, unaligned
from test_gpu_cfg_rescale import ulp_dist
from test_tcfg import product_schedule, reference_schedule

pytestmark = pytest.mark.gpu


# ---- the words pass ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("ps", [8, 104, 8192 + 16, 3 * 64 * 64, 7, 9, 8193])
def test_words_bit_exact(cuda_backend, dt, ps):
    gen = torch.Generator().manual_seed(ps)
    o = TCFGOracle()
    for layout in ("c", "cl") if ps % 64 == 0 else ("c",):
        a = _args(0, True, DT[dt], DT[dt], 3, ps, gen, layout=layout)
        w = cuda_backend.tcfg_words(a.e_cond, a.e_uncond)
        assert w.shape == (3, 2)
        assert torch.equal(w, cuda_backend.tcfg_words(a.e_cond, a.e_uncond)), "the words are not deterministic"
        same(w, o.tcfg_words(a.e_cond.cpu(), a.e_uncond.cpu()))
        for b in range(3):      # a sample alone, in fresh (differently aligned) storage, gives the same bits
            wb = cuda_backend.tcfg_words(a.e_cond[b:b + 1].clone(), a.e_uncond[b:b + 1].clone())
            assert torch.equal(wb[0], w[b])
    # unaligned storage takes the element-wise path: the same bits
    a = _args(0, True, DT[dt], DT[dt], 2, ps, gen)
    ec, eu = unaligned(a.e_cond), unaligned(a.e_uncond)
    same(cuda_backend.tcfg_words(ec, eu), o.tcfg_words(ec.cpu(), eu.cpu()))
    same(cuda_backend.tcfg_words(ec, eu), cuda_backend.tcfg_words(a.e_cond, a.e_uncond))


@pytest.mark.parametrize("Bn", [1, 2, 5, 17, 64])
def test_words_batch_sizes(cuda_backend, Bn):
    gen = torch.Generator().manual_seed(Bn)
    a = _args(0, True, torch.bfloat16, torch.bfloat16, Bn, 4 * 32 * 32, gen)
    same(cuda_backend.tcfg_words(a.e_cond, a.e_uncond), TCFGOracle().tcfg_words(a.e_cond.cpu(), a.e_uncond.cpu()))


def test_words_constructed_and_ieee_edges(cuda_backend):
    D = 1000
    c = torch.randn(7, D).cuda()
    u = torch.randn(7, D).cuda()
    u[0] = c[0]                         # c == u: (0.5, 0.5)
    c[1], u[1] = 0.0, 0.0               # both zero: (1, 0)
    c[2], u[2] = 0.0, 0.0
    c[2, 0], u[2, 1] = 3.0, 3.0         # orthogonal, equal norms: (1, 0)
    c[3], u[3] = 0.0, 0.0
    c[3, 0], u[3, 1] = 3.0, 2.0         # orthogonal, ||c|| > ||u||: (0, 0)
    u[4, 17] = float("inf")
    c[5, 3] = float("nan")
    w = cuda_backend.tcfg_words(c, u).cpu()
    assert w[0].tolist() == [0.5, 0.5] and w[1].tolist() == [1.0, 0.0] and w[2].tolist() == [1.0, 0.0]
    assert w[3].tolist() == [0.0, 0.0]
    assert torch.isnan(w[4]).all() and torch.isnan(w[5]).all() and torch.isfinite(w[6]).all()
    same(w, TCFGOracle().tcfg_words(c.cpu(), u.cpu()))


# ---- the step ----------------------------------------------------------------------------------------------------------

def _check_step(be, a, words=None):
    a.cfgzero_s = None
    a.tcfg_w = be.tcfg_words(a.e_cond, a.e_uncond) if words is None else words
    m, o = be.step(a)
    mw, ow = TCFGOracle().step(cpu(a))
    assert (m is None) == (mw is None) and (o is None) == (ow is None)
    if m is not None:
        same(m, mw)
    if o is not None:
        same(o, ow)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])      # whole packets per sample / tails and the generic kernel
def test_step_vs_executor(cuda_backend, pair, ps):
    gen = torch.Generator().manual_seed(ps)
    for form in range(7):
        for param in range(6):
            for px0 in (False, True):
                a = _args(param, px0, DT[pair[0]], DT[pair[1]], 5, ps, gen, form,
                          per_sample=(form + param) % 2 == 1)
                if (form + param) % 3 == 0:
                    a.out2 = torch.empty_like(a.x) if form else None
                    a.want_m_out = form == 0
                _check_step(cuda_backend, a)
                if a.out2 is not None:
                    same(a.out2, TCFGOracle().step(cpu(a))[1])


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


EDGE_WORDS = [0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -1e-40, 0.5, 1.0]


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])
def test_step_ieee_edges(cuda_backend, pair, ps):
    """step_edges operands in the halves and x, and words of 0, -0, +-inf, NaN and subnormals: every row matches the
    executor bit for bit."""
    md, sd = DT[pair[0]], DT[pair[1]]
    rng = np.random.default_rng(ps)
    gen = torch.Generator().manual_seed(5)
    Bn = 6
    for param in range(6):
        for form in (0, 1, 4):
            a = _args(param, param % 2 == 0, md, sd, Bn, ps, gen, form, per_sample=param % 2 == 1)
            flat = lambda t: t.float().cpu().numpy().reshape(-1)
            streams = {"ec": flat(a.e_cond), "eu": flat(a.e_uncond), "x": flat(a.xe)}
            scatter_edges(streams, {"ec": md, "eu": md, "x": sd}, rng, frac=0.3)
            put = lambda v, like: torch.from_numpy(v.reshape(like.shape).copy()).to(like.dtype).cuda()
            a.e_cond, a.e_uncond = put(streams["ec"], a.e_cond), put(streams["eu"], a.e_uncond)
            a.xe = put(streams["x"], a.xe)
            if form:
                a.x = a.xe
            words = np.array([[EDGE_WORDS[int(i)] for i in rng.integers(len(EDGE_WORDS), size=2)] for _ in range(Bn)],
                             np.float32)
            _check_step(cuda_backend, a, torch.from_numpy(words).cuda())


def test_step_launch_beyond_2_31_elements(cuda_backend):
    """One words pass and one step over 2^31 + 1003 elements (bf16, one sample: the element-wise paths) against separate
    torch CUDA ops: the words within 2 ulp of the closed form on torch's fp64 sums, the step bit for bit from the
    device's words."""
    from dpm_solver_b200.ops import StepArgs
    n = 2 ** 31 + 1003
    ch = 2 ** 28
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((1, n), generator=g, device="cuda", dtype=torch.bfloat16)
    ec = torch.randn((1, n), generator=g, device="cuda", dtype=torch.bfloat16)
    eu = torch.empty_like(ec)
    for k in range(0, n, ch):      # u = 0.5*c + 0.5*noise: well away from the degenerate A == C, B == 0
        sl = slice(k, k + ch)
        eu[:, sl] = (0.5 * ec[:, sl].float() + 0.5 * torch.randn(ec[:, sl].shape, generator=g, device="cuda")).to(
            torch.bfloat16)
    w = cuda_backend.tcfg_words(ec, eu)
    A = Bs = C = 0.0
    for k in range(0, n, ch):
        c64, u64 = ec[:, k:k + ch].double(), eu[:, k:k + ch].double()
        A += float((u64 * u64).sum())
        Bs += float((u64 * c64).sum())
        C += float((c64 * c64).sum())
        del c64, u64
    assert ulp_dist(w.cpu().numpy().reshape(-1), words_closed_form(A, Bs, C).reshape(-1)) <= 2
    a = StepArgs(form=1, n_model=2, x=x, xe=x, e_cond=ec, e_uncond=eu, param=4, predict_x0=True, guidance=W,
                 alpha_e=0.8, sigma_e=0.6, a=0.9, c0=-0.3, state_dtype=torch.bfloat16, per_sample=n, tcfg_w=w)
    _, out = cuda_backend.step(a)
    wu, wc = w[:, 0:1], w[:, 1:2]
    for k in range(0, n, ch):
        sl = slice(k, k + ch)
        us = eu[:, sl].float() * wu + ec[:, sl].float() * wc
        gg = us + W * (ec[:, sl].float() - us)
        x0 = (x[:, sl].float() - 0.6 * gg).to(torch.bfloat16).float()     # the buffered value, in the state dtype
        want = (0.9 * x[:, sl].float() + (-0.3) * x0).to(torch.bfloat16)
        assert torch.equal(out[:, sl], want), k


# ---- end to end --------------------------------------------------------------------------------------------------------

def net(x, t, c):
    """Products and sums only: the same bits on the CPU and on the GPU for fp32 inputs."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.45 * x + 0.05 * cc * x - 0.1 + 0.05 * cc


def blind(x, t, c):
    return 0.45 * x - 0.1


def wrap(mt, ns, device, w=W, model=net, B=2, **kw):
    import dpm_solver_b200 as new
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free",
                             condition=torch.ones(B, 1, device=device), unconditional_condition=torch.zeros(B, 1, device=device),
                             guidance_scale=w, tcfg=True, **kw)


def _runs(be, mt, device, solver, sd=None, shape=(2, 4, 16, 16), intermediates=False, **kw):
    """(first call, second call, fresh solver) of one configuration."""
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    old = _on(be)
    try:
        ns = product_schedule(mt)
        fn = wrap(mt, ns, device, B=shape[0])
        x = torch.randn(shape, generator=torch.Generator().manual_seed(0)).to(device)
        mk = (lambda: new.UniPC(fn, ns, state_dtype=sd, **kw)) if solver == "unipc" else \
            (lambda: new.DPM_Solver(fn, ns, state_dtype=sd, **kw))
        skw = dict(steps=6, order=2) if solver == "unipc" else dict(steps=6, order=3, method="singlestep")
        if intermediates:
            skw["return_intermediate"] = True
        s = mk()
        return [s.sample(x.clone(), **skw), s.sample(x.clone(), **skw), mk().sample(x.clone(), **skw)]
    finally:
        ops.set_backend(old)


@pytest.mark.parametrize("mt", ["noise", "v", "flow", "edm"])
@pytest.mark.parametrize("solver", ["dpm", "unipc"])
def test_sample_vs_executor(cuda_backend, mt, solver):
    ys = _runs(cuda_backend, mt, "cuda", solver)
    yw = _runs(TCFGOracle(), mt, "cpu", solver)[0]
    for y in ys:
        same(y, yw)
    # with intermediates
    yi = _runs(cuda_backend, mt, "cuda", solver, intermediates=True)[0]
    yiw = _runs(TCFGOracle(), mt, "cpu", solver, intermediates=True)[0]
    assert len(yi[1]) == len(yiw[1])
    same(yi[0], yiw[0])
    for a, b in zip(yi[1], yiw[1]):
        same(a, b)
    # bf16 state: the network itself then computes in bf16, where torch's CPU and CUDA kernels round a python scalar
    # differently; the three device runs are bit-identical and the executor's run is within bf16 rounding
    ys = _runs(cuda_backend, mt, "cuda", solver, torch.bfloat16)
    yw = _runs(TCFGOracle(), mt, "cpu", solver, torch.bfloat16)[0].float()
    assert torch.equal(ys[0], ys[1]) and torch.equal(ys[0], ys[2])
    err = float((ys[0].float().cpu() - yw).abs().max() / yw.abs().max())
    assert err <= 2e-2, err
    yt = _runs(cuda_backend, mt, "cuda", solver, correcting_x0_fn="dynamic_thresholding")
    ytw = _runs(TCFGOracle(), mt, "cpu", solver, correcting_x0_fn="dynamic_thresholding")[0]
    for y in yt:
        same(y, ytw)


@pytest.mark.parametrize("mt", ["noise", "flow"])
def test_device_adaptive_controller_vs_executor(cuda_backend, mt):
    """The device controller runs its steps on dev_coef launches (the generic <PG> kernel): the run equals the one on a
    network that returns the TCFG output g, on the same controller."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    x = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(4)).cuda()
    kw = dict(order=2, method="adaptive", atol=0.05, rtol=0.1)
    y = new.DPM_Solver(wrap(mt, ns, "cuda"), ns).sample(x.clone(), **kw)
    g = guided_net(net, torch.zeros(2, 1), torch.ones(2, 1), W)     # (fp32 products and sums: the device's bits)

    def gnet(xx, tt):
        return g(xx.cpu(), tt.cpu()).to(xx.device)
    yg = new.DPM_Solver(new.model_wrapper(gnet, ns, model_type=mt), ns).sample(x.clone(), **kw)
    same(y, yg)


@pytest.mark.parametrize("mt", ["noise", "flow"])
def test_capture_replays_bit_identically(cuda_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    scales = torch.tensor([W, 2.0], device="cuda")
    s = new.DPM_Solver(wrap(mt, ns, "cuda", w=scales), ns)
    x = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(2)).cuda()
    skw = dict(steps=6, order=2)
    eager = s.sample(x.clone(), **skw)
    gr = s.capture(x, **skw)
    y1 = gr(x).clone()
    y2 = gr(x).clone()
    assert torch.equal(y1, y2) and torch.equal(y1, eager)
    # the scales are read in place: a rewrite takes effect at the next replay
    scales[1] = 7.0
    y3 = gr(x).clone()
    s2 = new.DPM_Solver(wrap(mt, ns, "cuda", w=torch.tensor([W, 7.0], device="cuda")), ns)
    assert torch.equal(y3, s2.sample(x.clone(), **skw)) and not torch.equal(y3, y1)


@pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")
@pytest.mark.parametrize("mt", ["noise", "x_start", "v", "score", "flow", "edm"])
def test_condition_blind_fp32_equals_the_reference_unguided_run(cuda_backend, mt):
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    shape = (4, 4, 64, 64)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1))
    ns = product_schedule(mt)
    y = new.DPM_Solver(wrap(mt, ns, "cuda", model=blind, B=4), ns).sample(x.cuda(), steps=6, order=2).cpu()
    rns = reference_schedule(mt)
    u = lambda xx, tt: blind(xx, tt, None)
    if mt in ("flow", "edm"):
        from flow_oracle import reference_solver as flow_solver
        from edm_oracle import reference_solver as edm_solver
        rs = (flow_solver if mt == "flow" else edm_solver)(u, rns, "dpmsolver++")
    else:
        rs = ref.DPM_Solver(ref.model_wrapper(u, rns, model_type=mt), rns, algorithm_type="dpmsolver++")
    yr = rs.sample(x, steps=6, order=2, method="multistep")
    assert torch.equal(y, yr), float((y - yr).abs().max())


@pytest.mark.parametrize("thr", [False, True])
def test_launch_counts(cuda_backend, thr):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    counts = {}
    for tc in (False, True):
        fn = new.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(2, 1).cuda(),
                               unconditional_condition=torch.zeros(2, 1).cuda(), guidance_scale=W, tcfg=tc)
        s = new.DPM_Solver(fn, ns, correcting_x0_fn="dynamic_thresholding" if thr else None)
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)    # plans, tables and prepared launches cached
        torch.cuda.synchronize()
        before = cuda_backend.launch_count()
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)
        counts[tc] = cuda_backend.launch_count() - before
    # 6 evaluations: +2 words launches each, +1 materialising launch each under thresholding
    assert counts[True] - counts[False] == 6 * (3 if thr else 2), counts
