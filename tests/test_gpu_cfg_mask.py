"""Regional classifier-free guidance on the H100: dpm_step_multi_masked against the numpy executor bit for bit on every
launch kind (dtype pairs, forms, parameterisations, K = 1..4, every map kind shared and per-sample, replicas, tails,
unaligned views, channels_last, dev_coef, tunings, IEEE edge operands and weights), against dpm_step_multi for maps of
ones, beyond 2^31 elements against separate torch ops, and sample() end to end against the executor and the
reference composition."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from cases import seeded
from cfg_mask_oracle import MaskOracle
from step_edges import assert_bits_equal, scatter_edges
from test_cfg_multi import SCALES as MULTI_SCALES, conds, reference_composed
from test_cfg_rescale import inner_net, schedules
from test_gpu_cfg_rescale import COEF, DT, PAIRS

pytestmark = pytest.mark.gpu

SCALES = {1: [5.0], 2: [7.5, -2.0], 3: [4.0, 0.0, -1.5], 4: [3.0, 1.0, -0.5, 0.0]}
# map kinds: None (ones), one weight per sample, a pixel map, a full element map; "s" shared by the batch, "b" per sample
KINDS = ("none", "p1s", "p1b", "pixs", "pixb", "els", "elb")


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 40 * 2 ** 30


def _offset(t, k=1):
    buf = torch.empty(t.numel() + k, dtype=t.dtype, device=t.device)
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


def _map(kind, B, C_, S, layout, gen):
    """A (w, period, sample_stride) map entry of `kind` for x of shape [B, C_, S] ('cl': [B, C_, S//4, 4])."""
    if kind == "none":
        return None
    per_sample = C_ * S
    rows = 1 if kind.endswith("s") else B
    period = {"p1": 1, "pi": S, "el": per_sample}[kind[:2]]
    if kind.startswith("pi") and layout == "cl":
        period = per_sample
    w = (torch.randint(-2, 7, (rows, period), generator=gen).float() * 0.25).cuda()
    return w, period, 0 if rows == 1 else period


def _masked_args(form, param, px0, md, sd, K, B, C_, S, gen, kinds, layout="c", dev_coef=False):
    from dpm_solver_b200.ops import StepArgs
    shape = (B, C_, S) if layout == "c" else (B, C_, S // 4, 4)

    def t(dtype, scale=1.0, shift=0.0):
        v = (torch.randn(shape, generator=gen) * scale + shift).to(dtype).cuda()
        return v.contiguous(memory_format=torch.channels_last) if layout == "cl" else v
    x = t(sd)
    ecs = tuple(t(md, 1.0 + 0.2 * k, 0.1 * k) for k in range(K))
    a = StepArgs(form=form, n_model=2, x=x if form else None, xe=x, e_cond=ecs[0], e_uncond=t(md), e_conds=ecs,
                 scales=tuple(SCALES[K]), param=param, predict_x0=px0, state_dtype=sd, want_m_out=True,
                 m1=t(sd) if form in (2, 3, 4, 5, 6) else None, m2=t(sd) if form in (3, 5, 6) else None,
                 per_sample=C_ * S, **COEF)
    a.masks = tuple(_map(kinds[k % len(kinds)], B, C_, S, layout, gen) for k in range(K))
    a.c0_on_old = form == 4 and param % 2 == 1
    if form:
        a.replicas = tuple(torch.full_like(x, float("nan")) for _ in range(K))
    if dev_coef:
        v = [COEF[k] for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e")]
        a.coef_dev = torch.tensor(v + [0.] * 5, dtype=torch.float32).cuda()
    return a


def _cpu(v):
    if torch.is_tensor(v):
        return v.cpu()
    if isinstance(v, tuple):
        return tuple(_cpu(e) for e in v)
    return v


def _check(be, a, thr=False, replicas=True):
    B = a.e_cond.shape[0]
    if thr:
        a.thr = (torch.rand(B, generator=torch.Generator().manual_seed(B)) * 2 + 0.5).cuda()
    if not replicas:
        a.replicas = None
    m, o = be.step(a)
    ac = dataclasses.replace(a, **{f.name: _cpu(getattr(a, f.name)) for f in dataclasses.fields(a)})
    ac.coef_dev, ac.replicas = None, None
    mw, ow = MaskOracle().step(ac)
    assert_bits_equal(m, mw, "m_out")
    if ow is not None:
        assert_bits_equal(o, ow, "out")
        for r in a.replicas or ():
            assert_bits_equal(r, o, "replica")


SHAPES = [(5, 3, 64), (5, 3, 37), (4, 8, 5)]     # packets with vector maps / tails and odd sizes / period 5 maps
PARAMS = [(0, False), (0, True), (1, True), (2, False), (3, True), (4, True), (4, False), (5, True)]


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_step_masked_vs_executor(cuda_backend, pair, shape, K):
    gen = torch.Generator().manual_seed(sum(shape) + K)
    md, sd = DT[pair[0]], DT[pair[1]]
    i = 0
    for form in range(7):
        for param, px0 in PARAMS:
            for thr in ((False, True) if px0 else (False,)):
                kinds = KINDS[i % len(KINDS):] + KINDS[:i % len(KINDS)]
                _check(cuda_backend, _masked_args(form, param, px0, md, sd, K, *shape, gen, kinds), thr,
                       replicas=i % 3 != 0)
                i += 1


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("K", [1, 4])
def test_step_masked_views_channels_last_dev_coef_tunings(cuda_backend, pair, K):
    gen = torch.Generator().manual_seed(7 + K)
    md, sd = DT[pair[0]], DT[pair[1]]
    try:
        for tuning in ((2, 0, 0), (2, 128, 1), (1, 0, 0), (2, 64, 2)):
            cuda_backend.set_tuning(*tuning)
            for form in range(7):
                for param in (0, 2, 4):
                    for kinds in (KINDS, KINDS[3:] + KINDS[:3]):
                        _check(cuda_backend, _masked_args(form, param, True, md, sd, K, 4, 8, 24, gen, kinds, "cl"),
                               True)
                        a = _masked_args(form, param, True, md, sd, K, 4, 3, 40, gen, kinds)
                        a.e_conds = tuple(_offset(e) for e in a.e_conds)
                        a.e_cond, a.e_uncond = a.e_conds[0], _offset(a.e_uncond)
                        _check(cuda_backend, a, param == 0)
                        b = _masked_args(form, param, True, md, sd, K, 4, 3, 64, gen, kinds)
                        b.masks = tuple(m if m is None else (_offset(m[0]), m[1], m[2]) for m in b.masks)
                        _check(cuda_backend, b, False)            # weights not 16-byte aligned: the generic kernel
                        if form:
                            _check(cuda_backend, _masked_args(form, param, True, md, sd, K, 4, 3, 64, gen, kinds,
                                                              dev_coef=True), False)
    finally:
        cuda_backend.set_tuning(2, 0, 0)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("K", [1, 3])
def test_step_masked_ieee_edges(cuda_backend, pair, K):
    """Edge operands scattered into every stream, and weights 0, -0, +-inf, NaN and subnormals in the maps."""
    rng = np.random.default_rng(K)
    gen = torch.Generator().manual_seed(K)
    md, sd = DT[pair[0]], DT[pair[1]]
    wedge = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-45, 1.0], np.float32)
    for form in (0, 1, 4, 5):
        for param, px0 in ((0, True), (0, False), (2, True), (4, True)):
            for kinds in (("elb", "pixs", "p1b", "els"), ("p1s", "elb", "none", "pixb")):
                a = _masked_args(form, param, px0, md, sd, K, 4, 3, 64, gen, kinds)
                streams = {"eu": a.e_uncond.float().cpu().numpy().reshape(-1)}
                dtypes = {"eu": md}
                for k, e in enumerate(a.e_conds):
                    streams["ec%d" % k], dtypes["ec%d" % k] = e.float().cpu().numpy().reshape(-1), md
                streams["x"], dtypes["x"] = a.xe.float().cpu().numpy().reshape(-1), sd
                scatter_edges(streams, dtypes, rng, frac=0.3)
                put = lambda v, like: torch.from_numpy(v.reshape(like.shape)).to(like.dtype).cuda()
                a.e_uncond = put(streams["eu"], a.e_uncond)
                a.e_conds = tuple(put(streams["ec%d" % k], e) for k, e in enumerate(a.e_conds))
                a.e_cond = a.e_conds[0]
                a.xe = put(streams["x"], a.xe)
                if form:
                    a.x = a.xe
                ms = []
                for m in a.masks:
                    if m is not None:
                        w = m[0].cpu().numpy().reshape(-1).copy()
                        idx = rng.choice(w.size, size=max(1, w.size // 4), replace=False)
                        w[idx] = wedge[rng.integers(len(wedge), size=idx.size)]
                        m = (torch.from_numpy(w.reshape(m[0].shape)).cuda(), m[1], m[2])
                    ms.append(m)
                a.masks = tuple(ms)
                _check(cuda_backend, a, px0 and param == 0)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
def test_maps_of_ones_equal_step_multi(cuda_backend, pair):
    gen = torch.Generator().manual_seed(3)
    md, sd = DT[pair[0]], DT[pair[1]]
    for K in (2, 3, 4):
        for form in range(7):
            for shape in ((5, 3, 64), (5, 3, 37)):
                a = _masked_args(form, 0, True, md, sd, K, *shape, gen, KINDS)
                a.masks = tuple(None if m is None else (torch.ones_like(m[0]), m[1], m[2]) for m in a.masks)
                m1, o1 = cuda_backend.step(a)
                reps = [r.clone() for r in a.replicas or ()]
                b = dataclasses.replace(a, masks=None)
                m2, o2 = cuda_backend.step(b)
                assert_bits_equal(m1, m2, "m_out")
                if o1 is not None:
                    assert_bits_equal(o1, o2, "out")
                    for r in reps:
                        assert_bits_equal(r, o2, "replica")


def test_capi_argument_errors_launch_nothing(cuda_backend):
    from dpm_solver_b200 import _lib
    L = _lib.lib()
    n = 64
    t = [torch.zeros(n, device="cuda") for _ in range(8)]
    d = _lib.StepDesc()
    d.x, d.xe, d.e_uncond, d.out, d.m1 = (v.data_ptr() for v in t[:5])
    d.n, d.per_sample, d.state_dtype, d.model_dtype, d.form, d.n_model, d.a, d.c0 = n, 16, 0, 0, 1, 2, 1.0, 1.0
    ec = (C.c_void_p * 4)(*[v.data_ptr() for v in t[4:8]])
    sc = (C.c_float * 4)(1.0, 2.0, 3.0, 4.0)
    w = torch.ones(16, device="cuda")
    maps = (_lib.CondMap * 4)(*[_lib.CondMap(w.data_ptr(), 16, 0)] * 4)
    before = L.dpm_launch_count()
    for n_cond in (0, 5, -1):
        assert L.dpm_step_multi_masked(C.byref(d), ec, sc, maps, n_cond, None, None) == -1
    assert L.dpm_step_multi_masked(C.byref(d), ec, sc, None, 2, None, None) == -1
    for period, stride in ((0, 0), (3, 0), (32, 0), (16, 8), (16, 1)):
        bad = (_lib.CondMap * 2)(_lib.CondMap(w.data_ptr(), 16, 0), _lib.CondMap(w.data_ptr(), period, stride))
        assert L.dpm_step_multi_masked(C.byref(d), ec, sc, bad, 2, None, None) == -1
    for ps in (0, 48):
        d.per_sample = ps
        assert L.dpm_step_multi_masked(C.byref(d), ec, sc, maps, 2, None, None) == -1
    d.per_sample = 16
    d.raw_round = 1
    assert L.dpm_step_multi_masked(C.byref(d), ec, sc, maps, 2, None, None) == -1
    torch.cuda.synchronize()
    assert L.dpm_launch_count() == before
    assert L.dpm_version() == 108        # an additive entry point: the version stays, the symbol is exported
    assert hasattr(L, "dpm_step_multi_masked")


@pytest.mark.parametrize("n,period", [(2 ** 31 + 1003, 1), (2 ** 31 + 1024, 2 ** 31 + 1024)])
def test_beyond_2g_elements_equals_torch_ops(cuda_backend, n, period):
    """One launch over more than 2^31 elements: bf16, LIN1 on eps, K = 1, a weight per sample (the generic kernel:
    samples of an odd size) or a full element map (the packet kernel); against separate torch ops in chunks."""
    from dpm_solver_b200.ops import StepArgs
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(1, n, generator=g, device="cuda", dtype=torch.bfloat16)
    eu = torch.randn(1, n, generator=g, device="cuda", dtype=torch.bfloat16)
    ec = torch.randn(1, n, generator=g, device="cuda", dtype=torch.bfloat16)
    w = torch.rand(1, period, generator=g, device="cuda") * 2 - 0.5
    a = StepArgs(form=1, n_model=2, x=x, e_cond=ec, e_uncond=eu, e_conds=(ec,), scales=(3.0,), masks=((w, period, 0),),
                 per_sample=n, state_dtype=torch.bfloat16, a=0.9, c0=-0.3)
    _, o = cuda_backend.step(a)
    del a
    step = 2 ** 28
    for s in range(0, n, step):
        e = min(n, s + step)
        wv = w[:, s:e] if period > 1 else w
        eps = eu[:, s:e].float() + (torch.tensor(3.0, device="cuda") * wv) * (ec[:, s:e].float() - eu[:, s:e].float())
        t0 = eps.to(torch.bfloat16).float()
        want = ((0.9 * x[:, s:e].float()) + (-0.3 * t0)).to(torch.bfloat16)
        assert_bits_equal(o[:, s:e], want, "chunk at %d" % s)


# ---- end to end --------------------------------------------------------------------------------------------------
SHAPE = (3, 4, 16, 16)
B = SHAPE[0]


def _masks(K, device, layout_kinds=("hw", "b1hw", "b111", "bchw")):
    g = torch.Generator().manual_seed(K)
    make = {"hw": (16, 16), "b1hw": (B, 1, 16, 16), "b111": (B, 1, 1, 1), "bchw": SHAPE}
    return [(torch.randint(0, 5, make[layout_kinds[k % 4]], generator=g).float() * 0.5).to(device) for k in range(K)]


def _wrap(ns, model_type, K, masks, device, net=None, scales=None):
    import dpm_solver_b200 as new
    return new.model_wrapper(net or inner_net(), ns, model_type=model_type, guidance_type="classifier-free",
                             condition=[c.to(device) for c in conds(K)],
                             unconditional_condition=torch.zeros(B, 1).to(device),
                             guidance_scale=scales or SCALES[K], guidance_mask=masks)


def _schedule(kind):
    import dpm_solver_b200 as new
    if kind == "flow":
        return new.NoiseScheduleFlow(shift=3.0), "flow"
    if kind == "edm":
        return new.NoiseScheduleEDM(), "edm"
    return schedules("sd")[2], kind


def _executor_run(kind, K, skw, solver_kw, x):
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    old = ops._backend
    ops.set_backend(MaskOracle())
    try:
        ns, mt = _schedule(kind)
        fn = _wrap(ns, mt, K, _masks(K, "cpu"), "cpu")
        return new.DPM_Solver(fn, ns, **solver_kw).sample(x.clone(), **skw)
    finally:
        ops.set_backend(old)


E2E = [("noise", 2, "multistep", 2, "dpmsolver++", True, None), ("v", 3, "singlestep", 3, "dpmsolver", False, None),
       ("x_start", 1, "singlestep_fixed", 2, "dpmsolver++", False, torch.bfloat16),
       ("flow", 4, "multistep", 3, "dpmsolver++", True, None), ("edm", 2, "multistep", 2, "dpmsolver++", False, None),
       ("flow", 2, "singlestep", 2, "dpmsolver", False, torch.bfloat16), ("score", 4, "multistep", 1, "dpmsolver", False,
                                                                         None)]


@pytest.mark.parametrize("case", E2E, ids=lambda c: "-".join(str(v) for v in c[:5]))
def test_sample_vs_executor(cuda_backend, case):
    """First and second call, a fresh solver, and intermediates: bit for bit the executor's run."""
    import dpm_solver_b200 as new
    kind, K, method, order, algo, thr, sd = case
    skw = dict(steps=6, order=order, method=method, skip_type="time_uniform")
    solver_kw = dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None, state_dtype=sd)
    x = seeded(SHAPE, 11)
    want = _executor_run(kind, K, skw, solver_kw, x)
    ns, mt = _schedule(kind)
    s = new.DPM_Solver(_wrap(ns, mt, K, _masks(K, "cuda"), "cuda"), ns, **solver_kw)
    for _ in range(2):
        assert_bits_equal(s.sample(x.cuda(), **skw), want, "sample")
    y, inter = new.DPM_Solver(_wrap(ns, mt, K, _masks(K, "cuda"), "cuda"), ns, **solver_kw).sample(
        x.cuda(), return_intermediate=True, **skw)
    assert_bits_equal(y, want, "fresh solver")
    assert_bits_equal(inter[-1], want, "last intermediate")


@pytest.mark.parametrize("K", [1, 3])
def test_adaptive_device_controller(cuda_backend, capsys, K):
    """The device controller: bit for bit the library's own run on the same eager-composed network with
    guidance_type="uncond" (w_k = fl32(s_k)*m_k, then eps_u + w_k*(eps_k - eps_u) in fp32 torch ops), same NFE."""
    import dpm_solver_b200 as new
    x = seeded(SHAPE, 4).cuda()
    akw = dict(order=2, method="adaptive", atol=0.05, rtol=0.1)
    _, _, pns = schedules("sd")
    masks = _masks(K, "cuda")
    capsys.readouterr()
    y = new.DPM_Solver(_wrap(pns, "noise", K, masks, "cuda"), pns).sample(x, **akw)
    nfe = int(capsys.readouterr().out.split()[-1])
    inner, n = inner_net(), K + 1
    c_in = torch.cat([torch.zeros(B, 1)] + conds(K)).cuda()
    ws = [torch.tensor(s, dtype=torch.float32, device="cuda") * m for s, m in zip(SCALES[K], masks)]

    def eager(xx, t_input):
        outs = inner(torch.cat([xx] * n), torch.cat([t_input] * n), c_in).chunk(n)
        e = outs[0]
        for w, ek in zip(ws, outs[1:]):
            e = e + w * (ek - outs[0])
        return e
    y_u = new.DPM_Solver(new.model_wrapper(eager, pns, guidance_type="uncond"), pns).sample(x, **akw)
    nfe_u = int(capsys.readouterr().out.split()[-1])
    assert nfe == nfe_u and torch.equal(y, y_u)


@pytest.mark.parametrize("thr", [False, True])
def test_capture_equals_eager_and_sees_rewritten_masks(cuda_backend, thr):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    masks = _masks(2, "cuda", ("b1hw", "b111"))        # canonical: read in place
    s = new.DPM_Solver(_wrap(pns, "noise", 2, masks, "cuda"), pns,
                       correcting_x0_fn="dynamic_thresholding" if thr else None)
    x = seeded(SHAPE, 2).cuda()
    skw = dict(steps=6, order=2, method="multistep")
    g = s.capture(x, **skw)
    assert torch.equal(g(x).clone(), s.sample(x.clone(), **skw))
    masks[0].mul_(0.5).add_(0.25)
    masks[1].neg_()
    got = g(x).clone()
    fresh = new.DPM_Solver(_wrap(pns, "noise", 2, [m.clone() for m in masks], "cuda"), pns,
                           correcting_x0_fn="dynamic_thresholding" if thr else None)
    assert torch.equal(got, fresh.sample(x.clone(), **skw))


@pytest.mark.parametrize("K", [2, 4])
def test_sample_fp32_masks_of_ones_vs_reference(cuda_backend, K):
    """fp32 [4,4,64,64], masks of ones: bit for bit the reference composition of the unmasked multi-condition run."""
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    shape = (4, 4, 64, 64)
    x = seeded(shape, 11)
    ones = [torch.ones(64, 64, device="cuda"), torch.ones(4, 1, 1, 1, device="cuda"), None,
            torch.ones(shape, device="cuda")][:K]
    for mt, algo, thr in (("noise", "dpmsolver++", True), ("v", "dpmsolver", False)):
        fn = new.model_wrapper(inner_net(), pns, model_type=mt, guidance_type="classifier-free",
                               condition=[c.cuda() for c in conds(K, 4)],
                               unconditional_condition=torch.zeros(4, 1).cuda(), guidance_scale=MULTI_SCALES[K],
                               guidance_mask=ones)
        skw = dict(steps=8, order=2, method="multistep", skip_type="time_uniform")
        yp = new.DPM_Solver(fn, pns, algorithm_type=algo,
                            correcting_x0_fn="dynamic_thresholding" if thr else None).sample(x.cuda(), **skw)
        ref, rns, composed = reference_composed(mt, K, MULTI_SCALES[K], batch=4)
        yr = ref.DPM_Solver(composed, rns, algorithm_type=algo,
                            correcting_x0_fn="dynamic_thresholding" if thr else None).sample(x.clone(), **skw)
        assert yp.cpu().numpy().tobytes() == yr.numpy().tobytes(), (mt, K)


def test_launch_counts(cuda_backend):
    """One fused launch per evaluation and one replicate per run, as without masks."""
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    s = new.DPM_Solver(_wrap(pns, "noise", 3, _masks(3, "cuda"), "cuda"), pns)
    x = seeded(SHAPE, 3).cuda()
    s.sample(x, steps=6, order=2)
    torch.cuda.synchronize()
    n0 = cuda_backend.launch_count()
    s.sample(x, steps=6, order=2)
    torch.cuda.synchronize()
    assert cuda_backend.launch_count() - n0 == 1 + 6
