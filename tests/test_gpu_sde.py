"""SDE-DPM-Solver++ on the H100: dpm_step_sde bit for bit against the numpy executor (tests/sde_oracle.py) with z drawn
by the contract, the in-kernel normals against torch's normal_ at the edges of ATen's launch geometry (and beyond
2^29 elements), sample() against the executor run, capture() replays and one full-size launch."""
import dataclasses
import random

import pytest
import torch

from sde_oracle import SdeOracle

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
PAIRS = [("f32", "f32"), ("bf16", "bf16"), ("f16", "f16"), ("bf16", "f32"), ("f16", "f32"), ("f32", "bf16")]


def gen(seed):
    return torch.Generator("cuda").manual_seed(seed)


def _G(n):
    """ATen's 256*grid of a normal_ over n fp32 elements on this device."""
    p = torch.cuda.get_device_properties(0)
    return 256 * min(p.multi_processor_count * (p.max_threads_per_multi_processor // 256), (n + 255) // 256)


def _launch(args, seed, be):
    from dpm_solver_b200 import ops
    g = gen(seed)
    args.sde = ops.SdeNoise(args.sde.cz, g)
    r = be.step(args)
    return r, g.get_offset()


@pytest.mark.parametrize("n", ["G-1", "G", "G+1", "4*G-1", "4*G+3", "4*G*5+17", 1000, 77, 8 * 270336 + 5])
def test_normals_equal_torch(n):
    """cz = 1 with a zero update: out is the noise itself, equal to normal_ bit for bit; the generator advances as
    normal_ advances it."""
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_LIN1
    if isinstance(n, str):
        G = _G(1 << 30)
        n = eval(n, {"G": G})
    x = torch.zeros(n, device="cuda")
    a = ops.StepArgs(form=FORM_LIN1, n_model=0, x=x, m0=x, a=0.0, c0=0.0, sde=ops.SdeNoise(1.0))
    (_, out), off = _launch(a, 123, ops.backend())
    g = gen(123)
    z = torch.empty(n, device="cuda").normal_(generator=g)
    assert torch.equal(out, z)
    assert off == g.get_offset()


def test_normals_beyond_2_29():
    """ATen splits a draw beyond 2^29 elements into launches of their own; the odd halves take the element path."""
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_LIN1
    n = (1 << 29) + 4099
    x = torch.zeros(n, device="cuda")
    a = ops.StepArgs(form=FORM_LIN1, n_model=0, x=x, m0=x, a=0.0, c0=0.0, sde=ops.SdeNoise(1.0))
    (_, out), off = _launch(a, 7, ops.backend())
    del a
    g = gen(7)
    z = torch.empty(n, device="cuda").normal_(generator=g)
    assert torch.equal(out, z)
    assert off == g.get_offset()


def _sized_shape(rng, n):
    """A [B, C, 1, W] shape of exactly n elements: B and C drawn from the divisors of n in 1..4 (C > 1, when n has
    one, so that channels_last is another storage order)."""
    B = rng.choice([b for b in (1, 2, 3, 4) if n % b == 0])
    Cs = [c for c in (3, 4, 2) if (n // B) % c == 0 and n // B // c > 1]
    C = rng.choice(Cs) if Cs else 1
    return (B, C, 1, n // (B * C))


def _case(rng, i, n=None):
    """One random launch: dtypes, outputs, form, guidance kind, thresholds, size and layout. `n`: the launch's number
    of elements (a [B, C, 1, W] shape), else a small [B, C, H, H] one."""
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2, FORM_LIN1, FORM_MS3, PARAM_NOISE, PARAM_V, PARAM_X_START
    md, sd = rng.choice(PAIRS)
    md, sd = DT[md], DT[sd]
    ne = rng.choice([0, 1, 2, 2])
    form = rng.choice([FORM_LIN1, FORM_DIFF2, FORM_MS3])
    if n is None:
        B = rng.choice([1, 2, 3])
        C = rng.choice([3, 4])
        H = rng.choice([5, 8, 16, 33])
        shape = (B, C, H, H)
    else:
        shape = _sized_shape(rng, n)
        B = shape[0]
    numel = shape[0] * shape[1] * shape[2] * shape[3]
    cl = rng.random() < 0.2
    unaligned = rng.random() < 0.15

    def t(dtype):
        v = torch.randn((numel + (1 if unaligned else 0)), device="cuda").to(dtype)
        v = v[1:] if unaligned else v
        v = v.view(shape)
        return v.contiguous(memory_format=torch.channels_last) if cl and not unaligned else v

    a = ops.StepArgs(form=form, n_model=ne, state_dtype=sd, x=t(sd))
    a.a, a.c0, a.c1, a.c2 = 0.93, 0.11, -0.27, 0.05
    a.w0, a.w1, a.w2, a.w3 = 1.3, 0.8, 0.6, 0.4
    if form in (FORM_DIFF2, FORM_MS3):
        a.m1 = t(sd)
    if form == FORM_MS3:
        a.m2 = t(sd)
    kind = "none"
    if ne == 0:
        a.m0 = t(sd)
    else:
        a.e_cond = t(md)
        a.param = rng.choice([PARAM_NOISE, PARAM_NOISE, PARAM_X_START, PARAM_V])
        a.predict_x0 = True
        a.alpha_e, a.sigma_e = 0.8, 0.6
        a.xe = a.x
        a.want_m_out = rng.random() < 0.7
        per_sample = numel // B
        if ne == 2:
            a.e_uncond = t(md)
            a.guidance = 3.5
            kind = rng.choice(["scalar", "per_sample", "rescale", "per_sample_rescale", "cfgzero", "tcfg"])
            gb = torch.tensor([rng.choice([1.0, 2.5, 4.0]) for _ in range(B)], device="cuda")
            if kind in ("per_sample", "per_sample_rescale"):
                a.guidance_b = gb
            if kind in ("rescale", "per_sample_rescale"):
                a.ratio, a.phi = torch.rand(B, device="cuda") + 0.5, 0.7
            if kind == "cfgzero":
                a.cfgzero_s = torch.rand(B, device="cuda")
                a.guidance_b = gb if rng.random() < 0.5 else None
            if kind == "tcfg":
                a.tcfg_w = torch.rand(B, 2, device="cuda")
            if kind != "scalar":
                a.per_sample = per_sample
            if rng.random() < 0.5 and not unaligned and not cl:
                a.out2 = torch.empty(shape, dtype=sd, device="cuda")
        if rng.random() < 0.3 and kind in ("none", "scalar"):
            a.per_sample = per_sample
            a.thr = torch.rand(B, device="cuda") + 0.5
    return a, kind


def _clone(a):
    import dataclasses
    b = dataclasses.replace(a)
    if a.out2 is not None:
        b.out2 = torch.empty_like(a.out2)
    return b


def test_launches_match_executor():
    from dpm_solver_b200 import ops
    rng = random.Random(2026)
    be, ex = ops.backend(), SdeOracle()
    seen = set()
    for i in range(160):
        a, kind = _case(rng, i)
        a.sde = ops.SdeNoise(0.37)
        b = _clone(a)
        (m_k, o_k), off_k = _launch(a, 1000 + i, be)
        (m_e, o_e), off_e = _launch(b, 1000 + i, ex)
        seen.add((a.form, a.n_model, kind))
        assert off_k == off_e
        assert torch.equal(o_k.float().contiguous(), o_e.float().contiguous()), (i, a.form, a.n_model, kind)
        if a.want_m_out and a.n_model:
            assert torch.equal(m_k.float().contiguous(), m_e.float().contiguous()), (i, kind)
        if a.out2 is not None:
            assert torch.equal(a.out2, o_k) and torch.equal(b.out2.float(), o_e.float())
    assert len(seen) >= 15


def _sizes(G):
    """Launch sizes around ATen's geometry: one element short of a round, one round, one element of lane 1, the last
    lane of round 0, round 1, round k, and sizes just past a multiple of G that are not multiples of 8 (a packet that
    crosses the segment's end)."""
    return [G - 1, G, G + 1, 4 * G - 1, 4 * G + 3, 4 * G * 2 + 17, 2 * G + 5, 3 * G + 1003, 5 * G + 7, 6 * G + 2]


def test_launches_at_the_edges_of_the_noise_geometry():
    """Random launches (every dtype pair, NE 0/1/2, every guidance kind, thresholds, out2, unaligned views and
    channels_last) at sizes whose noise reaches lanes 1-3 of each curand_normal4, rounds k >= 1 and packets that cross
    the segment's end, each with a model stage: bit for bit against the executor, generator offset included."""
    from dpm_solver_b200 import ops
    G = _G(1 << 30)
    sizes = _sizes(G)
    assert all(n > G for n in sizes[2:]) and any(n % 8 for n in sizes)
    rng = random.Random(2027)
    be = ops.backend()
    seen, staged = set(), set()
    for i in range(3 * len(sizes)):
        n = sizes[i % len(sizes)]
        a, kind = _case(rng, i, n)
        while i < len(sizes) and a.n_model == 0:
            a, kind = _case(rng, i, n)          # (the first pass over the sizes: each with a model stage)
        a.sde = ops.SdeNoise(0.37)
        b = _clone(a)
        (m_k, o_k), off_k = _launch(a, 3000 + i, be)
        (m_e, o_e), off_e = _launch(b, 3000 + i, SdeOracle())
        seen.add((a.n_model, kind, a.thr is not None, a.out2 is not None))
        if a.n_model:
            staged.add(n)
        assert off_k == off_e, (i, n)
        assert torch.equal(o_k.float().contiguous(), o_e.float().contiguous()), (i, n, a.form, a.n_model, kind)
        if a.want_m_out and a.n_model:
            assert torch.equal(m_k.float().contiguous(), m_e.float().contiguous()), (i, n, kind)
        if a.out2 is not None:
            assert torch.equal(a.out2, o_k) and torch.equal(b.out2.float(), o_e.float())
        del a, b, m_k, o_k, m_e, o_e
    kinds = {k for ne, k, _, _ in seen if ne == 2}
    assert kinds == {"scalar", "per_sample", "rescale", "per_sample_rescale", "cfgzero", "tcfg"}, kinds
    assert any(thr for _, _, thr, _ in seen) and any(o2 for _, _, _, o2 in seen)
    assert staged == set(sizes), "sizes without a launch that has a model stage: %s" % sorted(set(sizes) - staged)


@pytest.mark.parametrize("view", ["strided", "permuted"])
def test_x_in_neither_layout_takes_the_torch_drawn_noise(view):
    """x neither row-major nor channels_last: the launch runs row-major on copies, its noise drawn by torch on an
    empty_like of x (in x's own storage order) -- the contract's draw, which the executor makes."""
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2, PARAM_NOISE
    B, C, H, W = 2, 3, 40, 24
    if view == "strided":
        mk = lambda: torch.randn(B, C, H, 2 * W, device="cuda")[..., ::2]
    else:
        mk = lambda: torch.randn(B, H, C, W, device="cuda").permute(0, 2, 1, 3)
    x, m1, ec, eu = mk(), mk(), mk(), mk()
    assert ops.CudaBackend._layout(x) is None
    for ne in (0, 2):
        a = ops.StepArgs(form=FORM_DIFF2, n_model=ne, x=x, m1=m1, a=0.9, c0=0.1, c1=-0.2, w0=1.1, sde=ops.SdeNoise(0.3))
        if ne:
            a.e_cond, a.e_uncond, a.xe, a.predict_x0, a.param = ec, eu, x, True, PARAM_NOISE
            a.alpha_e, a.sigma_e, a.guidance, a.want_m_out = 0.8, 0.6, 7.5, True
        else:
            a.m0 = ec
        b = dataclasses.replace(a)
        ex = SdeOracle()
        (m_k, o_k), off_k = _launch(a, 11 + ne, ops.backend())
        (m_e, o_e), off_e = _launch(b, 11 + ne, ex)
        g = gen(11 + ne)
        z = torch.empty_like(x, dtype=torch.float32).normal_(generator=g)
        assert torch.equal(ex.draws[-1], z.cpu()) and off_k == off_e == g.get_offset()
        assert torch.equal(o_k, o_e.to(o_k.device)), view
        if ne:
            assert torch.equal(m_k, m_e.to(m_k.device))


def _sample(be, x, seed, state_dtype, order, eta, **kw):
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper, ops
    old = ops._backend
    ops.set_backend(be)
    try:
        ns = NoiseScheduleVP("discrete", betas=torch.linspace(1e-4, 2e-2, 1000))
        fn = model_wrapper(lambda x, t: 0.3 * torch.sin(x) + 0.2 * x, ns, model_type="noise")
        s = DPM_Solver(fn, ns, algorithm_type="sde-dpmsolver++", state_dtype=state_dtype)
        return s.sample(x, steps=7, order=order, eta=eta, generator=gen(seed), **kw)
    finally:
        ops.set_backend(old)


@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
def test_sample_matches_executor(state_dtype):
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper, ops
    x = torch.randn(3, 4, 16, 16, device="cuda")
    ns = NoiseScheduleVP("discrete", betas=torch.linspace(1e-4, 2e-2, 1000))
    fn = model_wrapper(lambda x, t: 0.3 * torch.sin(x) + 0.2 * x, ns, model_type="noise")
    s = DPM_Solver(fn, ns, algorithm_type="sde-dpmsolver++", state_dtype=state_dtype)     # one solver, reused
    for order, eta, st in ((1, 1.0, "dpmsolver"), (2, 0.5, "dpmsolver"), (2, 1.0, "taylor"), (3, 2.0, "taylor")):
        got = s.sample(x, steps=7, order=order, eta=eta, solver_type=st, generator=gen(order))
        want = _sample(SdeOracle(), x, order, state_dtype, order, eta, solver_type=st)
        assert torch.equal(got.float(), want.float().to(got.device)), (order, eta)


def test_capture_replays_the_eager_run():
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper
    ns = NoiseScheduleVP("discrete", betas=torch.linspace(1e-4, 2e-2, 1000))
    fn = model_wrapper(lambda x, t: 0.3 * torch.sin(x) + 0.2 * x, ns, model_type="noise")
    s = DPM_Solver(fn, ns, algorithm_type="sde-dpmsolver++")
    x = torch.randn(2, 4, 16, 16, device="cuda")
    g = gen(77)
    kw = dict(steps=6, order=2, eta=1.0, generator=g)
    replay = s.capture(x, **kw)
    state = g.get_state()
    off0 = g.get_offset()
    y1 = replay(x).clone()
    off1 = g.get_offset()
    y2 = replay(x).clone()
    assert off1 > off0 and g.get_offset() > off1
    assert not torch.equal(y1, y2)
    g.set_state(state)
    eager = s.sample(x, **kw)
    assert torch.equal(eager, y1)


def test_full_size_launch():
    """c2's bf16 [4096, 4, 64, 64] 2M update, once with one output and once with CFG, checked on slices."""
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2
    shape = (4096, 4, 64, 64)
    bf = torch.bfloat16
    x, m1, ec, eu = (torch.randn(shape, device="cuda").to(bf) for _ in range(4))
    for ne in (1, 2):
        a = ops.StepArgs(form=FORM_DIFF2, n_model=ne, x=x, xe=x, m1=m1, e_cond=ec, e_uncond=eu if ne == 2 else None,
                         predict_x0=True, alpha_e=0.8, sigma_e=0.6, guidance=7.5, a=0.9, c0=0.1, c1=-0.2, w0=1.1,
                         want_m_out=True, sde=ops.SdeNoise(0.3))
        (m, out), _ = _launch(a, 5, ops.backend())
        z = torch.empty(shape, device="cuda").normal_(generator=gen(5))
        for sl in (slice(0, 3), slice(2047, 2049), slice(4093, 4096)):
            ex = SdeOracle()
            b = ops.StepArgs(form=FORM_DIFF2, n_model=ne, x=x[sl], xe=x[sl], m1=m1[sl], e_cond=ec[sl],
                             e_uncond=eu[sl] if ne == 2 else None, predict_x0=True, alpha_e=0.8, sigma_e=0.6,
                             guidance=7.5, a=0.9, c0=0.1, c1=-0.2, w0=1.1, want_m_out=True, sde=ops.SdeNoise(0.3))
            # the slice's noise is the full draw's slice: stand it in for the executor's own draw
            ex_draw = z[sl].clone()
            orig = torch.Tensor.normal_
            try:
                torch.Tensor.normal_ = lambda self, generator=None: self.copy_(ex_draw)
                mo, oo = ex.step(b)
            finally:
                torch.Tensor.normal_ = orig
            assert torch.equal(out[sl], oo) and torch.equal(m[sl], mo)
