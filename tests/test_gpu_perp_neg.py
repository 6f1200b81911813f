"""Perp-Neg on the H100: dpm_perpneg_words bit for bit against the executor's exact summation order (every dtype, K,
sample size, layout, unaligned views, IEEE edges), deterministic and independent of batch position, one launch beyond
2^31 elements; sample() against the executor on the first and second call of one solver, the device adaptive
controller, capture() replay, full size, and the condition-blind identity against the unmodified reference."""
import numpy as np
import pytest
import torch

from oracle import ref_loader
from perpneg_oracle import PerpNegOracle, fold_order_case, words_exact
from test_gpu_cfg_zero_star import DT, _on, same, unaligned
from test_tcfg import product_schedule, reference_schedule

pytestmark = pytest.mark.gpu
SCALES = {2: [7.5, -3.0], 3: [5.0, -2.0, -1.5], 4: [4.0, -1.0, -0.5, -2.5]}


def _blocks(Bn, ps, K, dtype, gen, layout="c"):
    """u and K conditional outputs [Bn, ps] on the device (channels_last: [Bn, ps/64, 8, 8] in that format)."""
    u = torch.randn(Bn, ps, generator=gen)
    es = [u + (0.3 + k) * torch.randn(Bn, ps, generator=gen) + 0.2 * k * u for k in range(K)]
    out = []
    for t in [u] + es:
        t = t.to(dtype).cuda()
        if layout == "cl":
            t = t.reshape(Bn, ps // 64, 8, 8).contiguous(memory_format=torch.channels_last)
        out.append(t)
    return out[0], out[1:]


def _oracle(u, es, K):
    return PerpNegOracle().perpneg_words(u.cpu(), [e.cpu() for e in es], SCALES[K])


# ---- the words pass ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("K", [2, 3, 4])
@pytest.mark.parametrize("ps", [7, 9, 104, 8192 + 16, 8193, 3 * 64 * 64])
def test_words_bit_exact(cuda_backend, dt, K, ps):
    gen = torch.Generator().manual_seed(ps * 10 + K)
    for layout in ("c", "cl") if ps % 64 == 0 else ("c",):
        u, es = _blocks(3, ps, K, DT[dt], gen, layout)
        w = cuda_backend.perpneg_words(u, es, SCALES[K])
        assert w.shape == (3,) and w.dtype == torch.float32
        assert torch.equal(w, cuda_backend.perpneg_words(u, es, SCALES[K])), "the words are not deterministic"
        same(w, _oracle(u, es, K))
        for b in range(3):      # a sample alone, in fresh (differently aligned) storage, gives the same bits
            wb = cuda_backend.perpneg_words(u[b:b + 1].clone(), [e[b:b + 1].clone() for e in es], SCALES[K])
            assert torch.equal(wb[0], w[b])
    # unaligned storage takes the element-wise path: the same bits
    u, es = _blocks(2, ps, K, DT[dt], gen)
    uu, ue = unaligned(u), [unaligned(e) for e in es]
    same(cuda_backend.perpneg_words(uu, ue, SCALES[K]), cuda_backend.perpneg_words(u, es, SCALES[K]))
    same(cuda_backend.perpneg_words(uu, ue, SCALES[K]), _oracle(uu, ue, K))
    # one block unaligned is enough to leave the packet path
    ue2 = [es[0]] + [unaligned(e) for e in es[1:]]
    same(cuda_backend.perpneg_words(u, ue2, SCALES[K]), cuda_backend.perpneg_words(u, es, SCALES[K]))


@pytest.mark.parametrize("Bn", [1, 2, 5, 17, 64, 300])
def test_words_batch_sizes(cuda_backend, Bn):
    gen = torch.Generator().manual_seed(Bn)
    u, es = _blocks(Bn, 4 * 32 * 32, 2, torch.bfloat16, gen)
    same(cuda_backend.perpneg_words(u, es, SCALES[2]), _oracle(u, es, 2))


@pytest.mark.parametrize("dt", ["f32", "bf16", "f16"])
def test_words_ieee_edges(cuda_backend, dt):
    """Signed zeros, infinities, NaN and subnormals in every block, a sample with N == 0, perpendicular and exactly
    parallel negatives: bit for bit (NaN for NaN) against the executor."""
    D, K = 1000, 3
    gen = torch.Generator().manual_seed(7)
    u = torch.randn(10, D, generator=gen)
    es = [u + torch.randn(10, D, generator=gen) for _ in range(K)]
    tiny = {"f32": 1e-40, "bf16": 1e-39, "f16": 3e-6}[dt]
    es[0][0] = u[0]                                  # N == 0: w_1 = s_1
    u[1], es[0][1], es[1][1], es[2][1] = 0.0, 0.0, 0.0, 0.0
    es[0][1, :5], es[1][1, 5:9] = 1.0, -2.0          # perpendicular (disjoint) differences
    es[1][2] = u[2] + 2.0 * (es[0][2] - u[2])         # (nearly) parallel
    es[2][3, 17] = float("inf")
    u[4, 3] = float("-inf")
    es[0][5, 0] = float("nan")
    u[6] = -0.0
    es[0][6], es[1][6], es[2][6] = 0.0, -0.0, 0.0     # every block a zero of some sign: N == 0
    es[0][7, ::3] = tiny                             # subnormal differences
    u[7, 1::3] = -tiny
    es[1][8] = float("inf")                          # inf - inf in a difference
    u[8] = float("inf")
    blocks = [t.to(DT[dt]).cuda() for t in [u] + es]
    w = cuda_backend.perpneg_words(blocks[0], blocks[1:], SCALES[K])
    want = _oracle(blocks[0], blocks[1:], K)
    same(w, want)
    assert w[0] == np.float32(SCALES[K][0]) and w[6] == np.float32(SCALES[K][0])
    assert torch.isnan(w[3:6]).all() and torch.isnan(w[8])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_words_fold_order(cuda_backend, seed):
    """Blocks whose words move by hundreds of fp32 ulps when the fp64 fold s_1 - s_2*c_2 - ... runs in another order
    (perpneg_oracle.fold_order_case): bit for bit against the executor's left-to-right fold."""
    u, es, s = fold_order_case(seed=seed)
    w = cuda_backend.perpneg_words(torch.from_numpy(u).cuda(), [torch.from_numpy(e).cuda() for e in es], s)
    assert np.array_equal(w.cpu().numpy().view(np.uint32), words_exact(u, es, s).view(np.uint32))


def test_words_launch_beyond_2_31_elements(cuda_backend):
    """One words pass over 129 samples of 2^24 elements (2^31 + 2^24 in all, bf16, K = 2): sampled rows against the
    executor, bit for bit."""
    Bn, ps = 129, 2 ** 24
    g = torch.Generator(device="cuda").manual_seed(0)
    u = torch.randn((Bn, ps), generator=g, device="cuda", dtype=torch.bfloat16)
    es = [torch.randn((Bn, ps), generator=g, device="cuda", dtype=torch.bfloat16) for _ in range(2)]
    assert u.numel() > 2 ** 31
    w = cuda_backend.perpneg_words(u, es, SCALES[2]).cpu()
    for b in (0, 64, 128):
        rows = [t[b:b + 1].cpu() for t in [u] + es]
        want = words_exact(rows[0].float().numpy(), [r.float().numpy() for r in rows[1:]], SCALES[2])
        same(w[b:b + 1], torch.from_numpy(want))


# ---- end to end --------------------------------------------------------------------------------------------------------

def net(x, t, c):
    """Products and sums only, in fp32 (the same bits on the CPU and the GPU), returned in x's dtype; the conditional
    directions differ nonlinearly (no d_k is a multiple of d_1)."""
    xf = x.float()
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(torch.float32)
    return (0.45 * xf - 0.1 + 0.05 * cc * xf + 0.02 * cc * cc * xf * xf).to(x.dtype)


def blind(x, t, c):
    return 0.45 * x - 0.1


def conds(K, Bn, device):
    return [torch.full((Bn, 1), float(k + 1), device=device) for k in range(K)]


def wrap(mt, ns, device, K=2, model=net, B=2, scales=None, **kw):
    import dpm_solver_b200 as new
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free", condition=conds(K, B, device),
                             unconditional_condition=torch.zeros(B, 1, device=device),
                             guidance_scale=SCALES[K] if scales is None else scales, perp_neg=True, **kw)


def _runs(be, mt, device, K=3, sd=None, shape=(2, 4, 16, 16), intermediates=False, **kw):
    """(first call, second call, fresh solver) of one configuration."""
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    old = _on(be)
    try:
        ns = product_schedule(mt)
        fn = wrap(mt, ns, device, K, B=shape[0])
        x = torch.randn(shape, generator=torch.Generator().manual_seed(0)).to(device)
        mk = lambda: new.DPM_Solver(fn, ns, state_dtype=sd, **kw)
        skw = dict(steps=6, order=3, method="singlestep")
        if intermediates:
            skw["return_intermediate"] = True
        s = mk()
        return [s.sample(x.clone(), **skw), s.sample(x.clone(), **skw), mk().sample(x.clone(), **skw)]
    finally:
        ops.set_backend(old)


@pytest.mark.parametrize("mt", ["noise", "x_start", "v", "score", "flow", "edm"])
def test_sample_vs_executor(cuda_backend, mt):
    ys = _runs(cuda_backend, mt, "cuda")
    yw = _runs(PerpNegOracle(), mt, "cpu")[0]
    for y in ys:
        same(y, yw)
    yi = _runs(cuda_backend, mt, "cuda", intermediates=True)[0]
    yiw = _runs(PerpNegOracle(), mt, "cpu", intermediates=True)[0]
    assert len(yi[1]) == len(yiw[1])
    same(yi[0], yiw[0])
    for a, b in zip(yi[1], yiw[1]):
        same(a, b)
    yt = _runs(cuda_backend, mt, "cuda", K=2, correcting_x0_fn="dynamic_thresholding")
    ytw = _runs(PerpNegOracle(), mt, "cpu", K=2, correcting_x0_fn="dynamic_thresholding")[0]
    for y in yt:
        same(y, ytw)
    # bf16 state: the network returns bf16 computed in fp32, so both sides see the same outputs
    ys = _runs(cuda_backend, mt, "cuda", K=4, sd=torch.bfloat16)
    yw = _runs(PerpNegOracle(), mt, "cpu", K=4, sd=torch.bfloat16)[0]
    for y in ys:
        same(y, yw)


@pytest.mark.parametrize("mt", ["noise", "flow"])
def test_device_adaptive_controller(cuda_backend, mt):
    """The device controller runs its steps on dev_coef launches: the run equals the regional-guidance run on the same
    controller whose [B, 1, 1, 1] mask the network rewrites with the executor's words of its own outputs."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    K, s = 3, SCALES[3]
    x = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(4)).cuda()
    kw = dict(order=2, method="adaptive", atol=0.05, rtol=0.1)
    y = new.DPM_Solver(wrap(mt, ns, "cuda", K), ns).sample(x.clone(), **kw)
    mask = torch.ones(2, 1, 1, 1, device="cuda")

    def hooked(xx, tt, c):
        out = net(xx, tt, c)
        o = [b.cpu() for b in out.chunk(K + 1)]
        w = words_exact(o[0].reshape(2, -1).numpy(), [e.reshape(2, -1).numpy() for e in o[1:]], s)
        mask.copy_(torch.from_numpy(w).reshape(2, 1, 1, 1))
        return out
    import dpm_solver_b200 as new2
    fm = new2.model_wrapper(hooked, ns, model_type=mt, guidance_type="classifier-free", condition=conds(K, 2, "cuda"),
                            unconditional_condition=torch.zeros(2, 1, device="cuda"), guidance_scale=[1.0] + s[1:],
                            guidance_mask=[mask, None, None])
    ym = new.DPM_Solver(fm, ns).sample(x.clone(), **kw)
    same(y, ym)


@pytest.mark.parametrize("mt", ["noise", "flow"])
def test_capture_replays_bit_identically(cuda_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    s = new.DPM_Solver(wrap(mt, ns, "cuda", 2), ns, correcting_x0_fn="dynamic_thresholding")
    x = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(2)).cuda()
    skw = dict(steps=6, order=2)
    eager = s.sample(x.clone(), **skw)
    gr = s.capture(x, **skw)
    y1 = gr(x).clone()
    y2 = gr(x).clone()
    assert torch.equal(y1, y2) and torch.equal(y1, eager)
    x2 = torch.randn((2, 4, 16, 16), generator=torch.Generator().manual_seed(3)).cuda()
    assert torch.equal(gr(x2).clone(), s.sample(x2.clone(), **skw))


def test_full_size_bf16(cuda_backend):
    """K = 2 at bf16 [2048, 4, 64, 64]: the words bit for bit, and sample() against the executor."""
    shape = (2048, 4, 64, 64)
    gen = torch.Generator().manual_seed(11)
    u, es = _blocks(shape[0], 4 * 64 * 64, 2, torch.bfloat16, gen)
    same(cuda_backend.perpneg_words(u, es, SCALES[2]), _oracle(u, es, 2))
    del u, es
    y = _runs(cuda_backend, "noise", "cuda", K=2, sd=torch.bfloat16, shape=shape)
    yw = _runs(PerpNegOracle(), "noise", "cpu", K=2, sd=torch.bfloat16, shape=shape)[0]
    for v in y:
        same(v, yw)


@pytest.mark.parametrize("thr", [False, True])
def test_launch_counts(cuda_backend, thr):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    counts = {}
    for pn in (False, True):
        fn = new.model_wrapper(net, ns, guidance_type="classifier-free", condition=conds(2, 2, "cuda"),
                               unconditional_condition=torch.zeros(2, 1).cuda(), guidance_scale=SCALES[2],
                               perp_neg=pn)
        s = new.DPM_Solver(fn, ns, correcting_x0_fn="dynamic_thresholding" if thr else None)
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)
        torch.cuda.synchronize()
        before = cuda_backend.launch_count()
        s.sample(torch.randn(2, 4, 16, 16).cuda(), steps=6, order=2)
        counts[pn] = cuda_backend.launch_count() - before
    assert counts[True] - counts[False] == 6 * 2, counts


@pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")
@pytest.mark.parametrize("mt", ["noise", "x_start", "v", "score", "flow", "edm"])
def test_condition_blind_fp32_equals_the_reference_unguided_run(cuda_backend, mt):
    import dpm_solver_b200 as new
    ref = ref_loader.load("dpm_solver_pytorch")
    shape = (4, 4, 64, 64)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1))
    ns = product_schedule(mt)
    y = new.DPM_Solver(wrap(mt, ns, "cuda", 3, model=blind, B=4), ns).sample(x.cuda(), steps=6, order=2).cpu()
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
