"""Regional classifier-free guidance (`model_wrapper(..., condition=[c1, ..., cK], guidance_mask=[m1, ..., mK])`) on the
CPU: the product's host logic, driven by the numpy executor with dpm_step_multi_masked, against the UNMODIFIED reference
composed the way a user would compose it: each term from the reference's own model_wrapper for its condition at
guidance_scale=1, combined as eps_u + (s_k*m_k)*(eps_k - eps_u) in eager fp32 torch, and the reference DPM_Solver run on
that as a noise model."""
import os
from unittest import mock

import numpy as np
import pytest
import torch

from cases import seeded
from cfg_mask_oracle import MaskOracle
from test_cfg_multi import ALGOS, MODELS, conds
from test_cfg_rescale import inner_net, schedules

f32 = np.float32
B, C, H, W = 3, 2, 4, 4
SHAPE = (B, C, H, W)
SCALES = {1: [5.0], 2: [7.5, -2.0], 3: [4.0, 0.0, -1.5], 4: [3.0, 1.0, -0.5, 0.0]}


def _vals(shape, seed):
    """Mask values: fp32 numbers in [0, 1.5] with exact zeros and ones among them."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randint(0, 7, shape, generator=g).float() * 0.25
    return v


# one mask per shape class; the row-major period each one takes
MASKS = {
    "hw": (lambda: _vals((H, W), 1), H * W),
    "11hw": (lambda: _vals((1, 1, H, W), 2), H * W),
    "b1hw": (lambda: _vals((B, 1, H, W), 3), H * W),
    "bchw": (lambda: _vals((B, C, H, W), 4), C * H * W),
    "b111": (lambda: _vals((B, 1, 1, 1), 5), 1),
    "1c11": (lambda: _vals((1, C, 1, 1), 6), C * H * W),
}
KINDS = list(MASKS)


def masks_for(K, offset=0):
    """K masks of rotating shape classes (one entry None when K >= 3)."""
    ms = [MASKS[KINDS[(k + offset) % len(KINDS)]][0]() for k in range(K)]
    if K >= 3:
        ms[1] = None
    return ms


@pytest.fixture()
def mask_backend():
    from dpm_solver_b200 import ops
    be = MaskOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def _kw(algo, thr):
    return dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)


def product_fn(model_type, K, scales, masks, net=None, batch=B):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    return new.model_wrapper(net or inner_net(), pns, model_type=model_type, guidance_type="classifier-free",
                             condition=conds(K, batch), unconditional_condition=torch.zeros(batch, 1),
                             guidance_scale=scales, guidance_mask=masks), pns


def reference_composed(model_type, K, scales, masks, batch=B, net=None, sched="sd"):
    """model_fn(x, t_continuous) of the reference composition: w_k = fl32(s_k)*m_k, then eps_u + w_k*(eps_k - eps_u).
    `net(x, t, c)` (default inner_net) on the VP schedule `sched` of tests/golden/cases.make_betas."""
    ref, rns, _ = schedules(sched)
    uc = torch.zeros(batch, 1)
    fs = [ref.model_wrapper(net or inner_net(), rns, model_type=model_type, guidance_type="classifier-free", condition=c,
                            unconditional_condition=uc, guidance_scale=1.0) for c in [uc] + conds(K, batch)]
    ws = [torch.tensor(s, dtype=torch.float32) * (torch.ones(()) if m is None else m.float())
          for s, m in zip(scales, masks)]

    def composed(x, t):
        eu = fs[0](x, t)
        e = eu
        for w, f in zip(ws, fs[1:]):
            e = e + w * (f(x, t) - eu)
        return e
    return ref, rns, composed


FIXED = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2),
         ("singlestep", 3), ("singlestep_fixed", 2)]


@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("algo,thr", ALGOS)
@pytest.mark.parametrize("method,order", FIXED)
@pytest.mark.parametrize("model_type", MODELS)
def test_sample_matches_reference_composition(mask_backend, model_type, method, order, algo, thr, K):
    x = seeded(SHAPE, 11)
    masks = masks_for(K, offset=order + len(method))
    kw = dict(steps=6, order=order, method=method, skip_type="time_uniform",
              denoise_to_zero=model_type in ("noise", "v"), return_intermediate=True)
    fn, pns = product_fn(model_type, K, SCALES[K], masks)
    yp, ip = __import__("dpm_solver_b200").DPM_Solver(fn, pns, **_kw(algo, thr)).sample(x.clone(), **kw)
    ref, rns, composed = reference_composed(model_type, K, SCALES[K], masks)
    yr, ir = ref.DPM_Solver(composed, rns, **_kw(algo, thr)).sample(x.clone(), **kw)
    np.testing.assert_array_equal(yp.numpy(), yr.numpy())
    assert len(ip) == len(ir)
    for a, b in zip(ip, ir):
        np.testing.assert_array_equal(a.numpy(), b.numpy())
    assert any(e[0] == "masked" for e in mask_backend.log)


def _adaptive(solver, x, order):
    with mock.patch("builtins.print") as pr:
        y = solver.sample(x.clone(), order=order, method="adaptive", atol=0.05, rtol=0.1)
        return y, pr.call_args[0][-1]


@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("algo,thr", ALGOS)
@pytest.mark.parametrize("model_type,K", [("noise", 2), ("x_start", 3), ("v", 1), ("score", 4)])
def test_adaptive_matches_reference_composition(mask_backend, model_type, K, algo, thr, order):
    """The host controller: the same NFE, and the result within 1e-5 of the reference composition."""
    import dpm_solver_b200 as new
    x = seeded(SHAPE, 11)
    masks = masks_for(K, offset=K)
    ref, rns, composed = reference_composed(model_type, K, SCALES[K], masks)
    yr, nfe_r = _adaptive(ref.DPM_Solver(composed, rns, **_kw(algo, thr)), x, order)
    fn, pns = product_fn(model_type, K, SCALES[K], masks)
    yp, nfe_p = _adaptive(new.DPM_Solver(fn, pns, **_kw(algo, thr)), x, order)
    assert nfe_p == nfe_r
    err = np.abs(yp.numpy().astype(np.float64) - yr.numpy()).max() / max(np.abs(yr.numpy()).max(), 1e-30)
    assert err <= 1e-5


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_each_mask_shape(mask_backend, kind, channels_last):
    """Every shape class, on a row-major and a channels_last x: the canonical period (pixel maps become element maps
    in channels_last storage order) and the sampled result."""
    import dpm_solver_b200 as new
    make, period = MASKS[kind]
    m = make()
    if channels_last and period not in (1, C * H * W):
        period = C * H * W
    fn, pns = product_fn("v", 2, SCALES[2], [m, MASKS["hw"][0]()])
    x = seeded(SHAPE, 7)
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    w, p, stride = fn.cond_masks[0].weights(SHAPE, "cl" if channels_last else "c", x.device)
    assert p == period and stride in (0, p)
    assert stride == (p if m.dim() == 4 and m.shape[0] == B else 0)
    yp = new.DPM_Solver(fn, pns, **_kw("dpmsolver++", True)).sample(x.clone(), steps=5, order=2)
    ref, rns, composed = reference_composed("v", 2, SCALES[2], [m, MASKS["hw"][0]()])
    yr = ref.DPM_Solver(composed, rns, **_kw("dpmsolver++", True)).sample(x.clone(), steps=5, order=2)
    np.testing.assert_array_equal(yp.contiguous().numpy(), yr.contiguous().numpy())


def test_canonical_map_is_read_in_place(mask_backend):
    """A contiguous fp32 mask that already has its map's layout is read in place (so a captured graph sees rewrites);
    another form is converted once per version."""
    fn, _ = product_fn("noise", 2, SCALES[2], [torch.rand(B, 1, H, W), torch.rand(H, W, dtype=torch.float64)])
    w0, _, _ = fn.cond_masks[0].weights(SHAPE, "c", torch.device("cpu"))
    assert w0.data_ptr() == fn.cond_masks[0].mask.data_ptr()
    w1, _, _ = fn.cond_masks[1].weights(SHAPE, "c", torch.device("cpu"))
    assert w1.dtype == torch.float32 and w1.data_ptr() != fn.cond_masks[1].mask.data_ptr()
    assert fn.cond_masks[1].weights(SHAPE, "c", torch.device("cpu"))[0] is w1
    fn.cond_masks[1].mask.mul_(2)
    w2, _, _ = fn.cond_masks[1].weights(SHAPE, "c", torch.device("cpu"))
    assert torch.equal(w2, 2 * w1)


def _run(fn, pns, thr=False, **kw):
    import dpm_solver_b200 as new
    return new.DPM_Solver(fn, pns, **_kw("dpmsolver++", thr)).sample(seeded(SHAPE, 5), steps=5, order=2, **kw)


@pytest.mark.parametrize("thr", [False, True])
@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_masks_of_ones(mask_backend, K, thr):
    """Masks of ones equal the unmasked multi-condition run bit for bit (K >= 2) and the one-condition CFG run (K = 1,
    s != 1); at s == 1 the CFG run bypasses and the masked one combines."""
    import dpm_solver_b200 as new
    ones = [torch.ones(H, W), torch.ones(B, 1, 1, 1), None, torch.ones(SHAPE)][:K]
    fn, pns = product_fn("x_start", K, SCALES[K], ones)
    y = _run(fn, pns, thr)
    if K >= 2:
        plain, _ = product_fn("x_start", K, SCALES[K], None)
    else:
        _, _, pns = schedules("sd")
        plain = new.model_wrapper(inner_net(), pns, model_type="x_start", guidance_type="classifier-free",
                                  condition=conds(1)[0], unconditional_condition=torch.zeros(B, 1),
                                  guidance_scale=SCALES[1][0])
    np.testing.assert_array_equal(y.numpy(), _run(plain, pns, thr).numpy())


@pytest.mark.parametrize("K", [1, 2, 3])
def test_per_sample_weights_equal_rowwise_scales(mask_backend, K):
    """A [B,1,1,1] mask with scales 1 equals, row by row, the run with that row's scales."""
    import dpm_solver_b200 as new
    rows = torch.tensor([[2.5, -1.0, 0.0], [6.0, 0.5, 1.5], [0.25, 3.0, -2.0]])[:, :K]     # [B, K]
    fn, pns = product_fn("v", K, [1.0] * K, [rows[:, k].reshape(B, 1, 1, 1) for k in range(K)])
    y = _run(fn, pns)
    x = seeded(SHAPE, 5)
    for b in range(B):
        s = rows[b].tolist()
        if K == 1:
            one = new.model_wrapper(inner_net(), pns, model_type="v", guidance_type="classifier-free",
                                    condition=conds(1, 1)[0], unconditional_condition=torch.zeros(1, 1),
                                    guidance_scale=s[0])
        else:
            one, _ = product_fn("v", K, s, None, batch=1)
        yb = new.DPM_Solver(one, pns, **_kw("dpmsolver++", False)).sample(x[b:b + 1].clone(), steps=5, order=2)
        np.testing.assert_array_equal(y[b:b + 1].numpy(), yb.numpy())


@pytest.mark.parametrize("K", [1, 2, 4])
def test_direct_model_fn_call(mask_backend, K):
    """model_fn(x, t) is the masked combine, for one time label and for one label per sample."""
    x = seeded(SHAPE, 3)
    masks = masks_for(K, offset=2)
    for model_type in MODELS:
        fn, _ = product_fn(model_type, K, SCALES[K], masks)
        _, _, composed = reference_composed(model_type, K, SCALES[K], masks)
        for t in (torch.full((B,), 0.6), torch.linspace(0.9, 0.2, B)):
            np.testing.assert_array_equal(fn(x, t).numpy(), composed(x, t).numpy())


@pytest.mark.parametrize("thr", [False, True])
@pytest.mark.parametrize("K", [1, 3])
def test_launches_and_network_calls(mask_backend, K, thr):
    """As without masks: one network call per evaluation on (K+1)B rows, one fused launch per evaluation (plus the
    materialising launch and the quantile with thresholding) and one replicate launch per run."""
    calls = []
    inner = inner_net()

    def net(x, t, c):
        calls.append(tuple(x.shape))
        return inner(x, t, c)
    fn, pns = product_fn("noise", K, SCALES[K], masks_for(K), net=net)
    nfe = 5
    mask_backend.log.clear()
    n0 = mask_backend.launches
    _run(fn, pns, thr)
    log = list(mask_backend.log)
    assert calls == [((K + 1) * B,) + SHAPE[1:]] * nfe
    assert log.count(("replicate", K + 1)) == 1
    assert len([e for e in log if e[0] == "masked" and e[1] != 0]) == nfe
    if thr:
        assert log.count(("masked", 0)) == nfe and log.count(("quantile", 1)) == nfe
        assert mask_backend.launches - n0 == 1 + 3 * nfe
    else:
        assert ("masked", 0) not in log
        assert mask_backend.launches - n0 == 1 + nfe


# ---- batch sharding ------------------------------------------------------------------------------------------------------

def _sharded_masks():
    return [_vals((4, 1, H, W), 21), _vals((H, W), 22)]


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dpm_solver_b200 import ops
        import dpm_solver_b200 as new
        ops.set_backend(MaskOracle())
        rows = slice(2 * rank, 2 * rank + 2)
        m = _sharded_masks()
        fn, pns = product_fn("noise", 2, SCALES[2], [m[0][rows], m[1]], batch=2)
        x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))[rows]
        y = new.DPM_Solver(fn, pns, plan_broadcast=True).sample(x, steps=5, order=2)
        q.put((rank, y))
    finally:
        dist.destroy_process_group()


def test_batch_sharding(mask_backend):
    """Two gloo ranks of two samples each, the per-sample masks split like the batch, equal the unsharded run of four."""
    import socket
    import torch.multiprocessing as mp
    import dpm_solver_b200 as new
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    fn, pns = product_fn("noise", 2, SCALES[2], _sharded_masks(), batch=4)
    x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))
    y = new.DPM_Solver(fn, pns).sample(x, steps=5, order=2)
    assert torch.equal(torch.cat([got[0], got[1]]), y)


# ---- rejections ----------------------------------------------------------------------------------------------------------

def test_invalid_arguments_raise(mask_backend):
    import dpm_solver_b200 as new
    from dpm_solver_b200.unipc import UniPC
    _, _, pns = schedules("sd")
    calls = []
    net = inner_net(calls)
    uc = torch.zeros(B, 1)
    hw = torch.ones(H, W)
    n0 = mask_backend.launches

    def mk(cond=None, scale=(7.5, 2.0), masks=(hw, hw), **kw):
        kw.setdefault("guidance_type", "classifier-free")
        return new.model_wrapper(net, pns, condition=conds(2) if cond is None else cond,
                                 unconditional_condition=kw.pop("uc", uc), guidance_scale=scale, guidance_mask=masks,
                                 **kw)
    cases = [
        (dict(guidance_type="uncond"), "classifier-free"),
        (dict(uc=None), "unconditional_condition"),
        (dict(masks=[hw]), "1 guidance masks for 2"),
        (dict(masks=[hw, hw, hw]), "3 guidance masks for 2"),
        (dict(masks=[hw, 1.0]), "tensor or None"),
        (dict(cond=conds(1)[0], scale=torch.tensor([1.0, 2.0, 3.0]), masks=hw), "per-sample"),
        (dict(scale=torch.ones(B, 2)), "per-sample"),
        (dict(scale=[torch.ones(B), torch.ones(B)]), "per-sample"),
        (dict(guidance_rescale=0.7), "guidance_rescale"),
        (dict(apg_eta=0.0), "adaptive projected guidance"),
        (dict(cfg_zero_star=True), "cfg_zero_star"),
        (dict(cfg_pp=True), "cfg_pp"),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            mk(**kw)
    with pytest.raises(ValueError, match="reference_rounding"):
        new.DPM_Solver(mk(), pns, algorithm_type="dpmsolver", reference_rounding=True)
    with pytest.raises(ValueError, match="guidance_mask"):
        UniPC(mk(cond=conds(1), scale=[7.5], masks=[hw]), pns).sample(seeded(SHAPE, 1), steps=5)
    # shapes that do not broadcast to x, or a batch extent other than 1 or B: at the first evaluation, before any launch
    for bad in (torch.ones(H + 1, W), torch.ones(2, 1, H, W), torch.ones(B, C + 1, 1, 1), torch.ones(1, B, C, H, W)):
        fn = mk(masks=(hw, bad))
        with pytest.raises(ValueError, match="broadcast"):
            new.DPM_Solver(fn, pns).sample(seeded(SHAPE, 1), steps=5)
        with pytest.raises(ValueError, match="broadcast"):
            fn(seeded(SHAPE, 1), torch.full((B,), 0.5))
    assert calls == [] and mask_backend.launches == n0


def test_default_changes_nothing(mask_backend):
    """guidance_mask=None: no masked path runs."""
    fn, pns = product_fn("noise", 2, SCALES[2], None)
    assert fn.cond_masks is None
    mask_backend.log.clear()
    _run(fn, pns)
    assert not any(e[0] == "masked" for e in mask_backend.log)
