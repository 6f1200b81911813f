"""CFG++ (`model_wrapper(..., cfg_pp=True)`) on the CPU: the product's host logic on the numpy executor
(tests/cfgpp_oracle.py). A condition-blind network makes a CFG++ run the plain DPM-Solver++ run, checked by value
against the UNMODIFIED reference; a condition-aware one follows an fp64 transcription of the paper's recurrences; order 1
equals plain CFG with the per-step scale lambda/(1 - e^-h); per-sample rows, batch sharding and every rejection."""
import math
import os

import numpy as np
import pytest
import torch

from cases import make_betas
from cfgpp_oracle import CFGPPOracle, cfgpp_fp64
from oracle import ref_loader

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
B, SHAPE = 2, (2, 3, 6, 6)
MODEL_TYPES = ["noise", "x_start", "v", "score", "flow", "edm"]
SCALES = [0.3, 1.0, 7.5, "per_sample"]


@pytest.fixture()
def pp_backend():
    from dpm_solver_b200 import ops
    be = CFGPPOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def blind(x, t, c=None):
    """Blind to the condition, products and sums only (exact IEEE ops: the same bits for any batch layout)."""
    tt = t.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.45 * x + (0.05 * x) * x - 0.1 + 1e-4 * tt


def aware(x, t, c):
    """Depends on the condition: the guided and the unconditional predictions differ."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return blind(x, t) + 0.08 * cc * x - 0.05 * cc


def product_schedule(mt):
    import dpm_solver_b200 as new
    if mt == "flow":
        return new.NoiseScheduleFlow(shift=3.0)
    if mt == "edm":
        return new.NoiseScheduleEDM()
    return new.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def reference_solver(mt, net):
    """The unmodified reference's DPM-Solver++ on a single (unguided) network."""
    if mt == "flow":
        from flow_oracle import reference_schedule, reference_solver as rs
        return rs(net, reference_schedule(3.0), "dpmsolver++")
    if mt == "edm":
        from edm_oracle import reference_schedule, reference_solver as rs
        return rs(net, reference_schedule(), "dpmsolver++")
    ref = ref_loader.load("dpm_solver_pytorch")
    rns = ref.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    return ref.DPM_Solver(ref.model_wrapper(net, rns, model_type=mt), rns, algorithm_type="dpmsolver++")


def wrap(mt, ns, w, model=aware, n=B, **kw):
    import dpm_solver_b200 as new
    if w == "per_sample":
        w = torch.tensor([0.3, 1.0, 7.5, 0.6][:n])
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free", condition=torch.ones(n, 1),
                             unconditional_condition=torch.zeros(n, 1), guidance_scale=w, **kw)


def x_T(seed=0, shape=SHAPE):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed))


# ---- a condition-blind network: the plain DPM-Solver++ run, against the reference ---------------------------------------

@needs_ref
@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("w", SCALES, ids=str)
def test_condition_blind_equals_reference(pp_backend, mt, order, w):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    skw = dict(steps=6, order=order, method="multistep")      # steps < 10: lower_order_final lowers the last update
    y = new.DPM_Solver(wrap(mt, ns, w, model=blind, cfg_pp=True), ns).sample(x_T(), **skw)
    yr = reference_solver(mt, lambda x, t: blind(x, t)).sample(x_T(), **skw)
    assert torch.equal(y, yr), float((y - yr).abs().max())
    assert any(e[0] == "cfgpp" for e in pp_backend.log)


@needs_ref
@pytest.mark.parametrize("mt", ["noise", "v", "flow", "edm"])
@pytest.mark.parametrize("skip", ["time_uniform", "logSNR", "time_quadratic"])
@pytest.mark.parametrize("solver_type", ["dpmsolver", "taylor"])
@pytest.mark.parametrize("steps,lof", [(6, False), (12, True)])
def test_condition_blind_solver_and_skip_types(pp_backend, mt, skip, solver_type, steps, lof):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    skw = dict(steps=steps, order=2, method="multistep", skip_type=skip, solver_type=solver_type,
               lower_order_final=lof)
    y = new.DPM_Solver(wrap(mt, ns, 0.7, model=blind, cfg_pp=True), ns).sample(x_T(1), **skw)
    yr = reference_solver(mt, lambda x, t: blind(x, t)).sample(x_T(1), **skw)
    assert torch.equal(y, yr), float((y - yr).abs().max())


@needs_ref
@pytest.mark.parametrize("mt", ["noise", "x_start", "flow"])
@pytest.mark.parametrize("order", [1, 2])
def test_condition_blind_inverse_and_denoise(pp_backend, mt, order):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    skw = dict(steps=5, order=order, method="multistep")
    s = new.DPM_Solver(wrap(mt, ns, 2.0, model=blind, cfg_pp=True), ns)
    r = reference_solver(mt, lambda x, t: blind(x, t))
    y, yr = s.inverse(x_T(2), **skw), r.inverse(x_T(2), **skw)
    assert torch.equal(y, yr), float((y - yr).abs().max())
    y, yr = s.sample(x_T(2), denoise_to_zero=True, **skw), r.sample(x_T(2), denoise_to_zero=True, **skw)
    assert torch.equal(y, yr), float((y - yr).abs().max())


# ---- a condition-aware network: the fp64 transcription -------------------------------------------------------------------

def _fp64_run(mt, ns, w, order, solver_type, steps, x):
    """cfgpp_fp64 on the product's grid and fp32 marginals, the network evaluated in fp64."""
    from dpm_solver_b200 import DPM_Solver, plan as P
    s = DPM_Solver(wrap(mt, ns, w), ns)
    ts = s.get_time_steps("time_uniform", ns.T, 1. / ns.total_N, steps, "cpu")
    m = P.Marginals(ns, ts)
    lam, al, sg = (v.double().numpy() for v in (m.lam, m.alpha, m.sigma))
    fn = s._wrapped
    tin = fn.get_model_input_time(ts).double()

    def x0(out, xx, i):
        if mt == "noise":
            return (xx - sg[i] * out) / al[i]
        if mt == "v":
            return al[i] * xx - sg[i] * out
        return xx - sg[i] * out          # flow

    def pair(xx, i):
        xt = torch.from_numpy(xx)
        t = tin[i].expand(B)
        c, u = aware(xt, t, torch.ones(B, 1)).numpy(), aware(xt, t, torch.zeros(B, 1)).numpy()
        U, C = x0(u, xx, i), x0(c, xx, i)
        return U + w * (C - U), U
    return cfgpp_fp64(pair, lam, al, x.double().numpy(), order, solver_type), (lam, al, sg, pair)


@pytest.mark.parametrize("mt", ["noise", "v", "flow"])
@pytest.mark.parametrize("order,solver_type", [(1, "dpmsolver"), (2, "dpmsolver"), (2, "taylor")])
@pytest.mark.parametrize("w", [0.3, 1.0])
def test_condition_aware_follows_fp64_transcription(pp_backend, mt, order, solver_type, w):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    y = new.DPM_Solver(wrap(mt, ns, w, cfg_pp=True), ns).sample(x_T(3), steps=8, order=order, solver_type=solver_type)
    want, (lam, al, sg, pair) = _fp64_run(mt, ns, w, order, solver_type, 8, x_T(3))
    err = float(np.abs(y.double().numpy() - want).max() / np.abs(want).max())
    assert err <= 1e-5, err
    # the plain CFG run with the same scale is far from it: the test sees the guidance
    y0 = new.DPM_Solver(wrap(mt, ns, w), ns).sample(x_T(3), steps=8, order=order, solver_type=solver_type)
    assert float(np.abs(y0.double().numpy() - want).max() / np.abs(want).max()) > 1e-3
    if order == 1:
        # the paper's DDIM form, x_t = alpha_t*G + sigma_t*eps_u with eps_u = (x - alpha_s*U)/sigma_s, in fp64
        xx = x_T(3).double().numpy()
        for i in range(8):
            G, U = pair(xx, i)
            xx = al[i + 1] * G + sg[i + 1] * (xx - al[i] * U) / sg[i]
        err = float(np.abs(y.double().numpy() - xx).max() / np.abs(xx).max())
        assert err <= 1e-5, err


@pytest.mark.parametrize("mt", ["noise", "x_start", "v", "score", "flow", "edm"])
@pytest.mark.parametrize("w", [0.3, 0.8])
def test_order_one_is_plain_cfg_with_a_per_step_scale(pp_backend, mt, w):
    """Order-1 CFG++ with lambda is plain CFG whose scale at the step s -> t is lambda/(1 - e^-h): checked through a
    network that forms that guided output itself, independently of the kernel's op order."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    steps = 7
    s = new.DPM_Solver(wrap(mt, ns, w, cfg_pp=True), ns)
    y = s.sample(x_T(4), steps=steps, order=1)
    ts = s.get_time_steps("time_uniform", ns.T, 1. / ns.total_N, steps, "cpu")
    lam = ns.marginal_lambda(ts).double()
    tin = s._wrapped.get_model_input_time(ts)
    scale = {float(tin[i]): w / -math.expm1(-float(lam[i + 1] - lam[i])) for i in range(steps)}

    def per_step(x, t, c):
        u, cc = aware(x, t, torch.zeros(B, 1)), aware(x, t, torch.ones(B, 1))
        sv = scale[float(t.reshape(-1)[0])]
        return u + sv * (cc - u)        # (every parameterisation is affine in the output at a fixed state)
    plain = new.DPM_Solver(new.model_wrapper(lambda x, t: per_step(x, t, None), ns, model_type=mt), ns)
    y0 = plain.sample(x_T(4), steps=steps, order=1)
    err = float((y.double() - y0.double()).abs().max() / y0.double().abs().max())
    assert err <= 1e-5, err


# ---- per-sample rows, direct calls, buffers ------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_per_sample_rows_equal_their_scalar_runs(pp_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    ws = [0.6, 0.25, 1.0]
    kw = dict(steps=6, order=2)
    x = x_T(5, (3,) + SHAPE[1:])
    yb = new.DPM_Solver(wrap(mt, ns, torch.tensor(ws), n=3, cfg_pp=True), ns).sample(x, **kw)
    for b, w in enumerate(ws):
        yw = new.DPM_Solver(wrap(mt, ns, w, n=3, cfg_pp=True), ns).sample(x, **kw)
        if w != 1.0:
            assert torch.equal(yb[b:b + 1], yw[b:b + 1]), b
        else:
            # a per-sample 1 takes e_c, a scalar 1 combines u + 1*(c - u): the same to within an fp32 rounding
            assert torch.allclose(yb[b:b + 1], yw[b:b + 1], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("w", [0.3, 1.0, "per_sample"], ids=str)
def test_direct_calls_return_the_plain_guided_values(pp_backend, w):
    import dpm_solver_b200 as new
    ns = product_schedule("v")
    x, t = x_T(6), torch.full((B,), 0.5)
    calls = []

    def counted(xx, tt, cc):
        calls.append(xx.shape[0])
        return aware(xx, tt, cc)
    fn, f0 = wrap("v", ns, w, model=counted, cfg_pp=True), wrap("v", ns, w)
    assert torch.equal(fn(x, t), f0(x, t))
    assert calls == [B if w == 1.0 else 2 * B]          # a scalar 1 keeps the reference's bypass in a direct call
    # data_prediction_fn (and so denoise_to_zero) is the existing CFG path: G
    s, s0 = new.DPM_Solver(fn, ns), new.DPM_Solver(f0, ns)
    tt = torch.tensor([0.5])
    if w != 1.0:
        assert torch.equal(s.data_prediction_fn(x, tt), s0.data_prediction_fn(x, tt))


def test_the_buffer_holds_u_and_launches_are_fused(pp_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    pp_backend.log.clear()
    new.DPM_Solver(wrap("noise", ns, 0.5, cfg_pp=True), ns).sample(x_T(), steps=6, order=2)
    # one launch per evaluation, the run's first network input from dpm_duplicate
    assert pp_backend.log == [("cfgpp", 1)] + [("cfgpp", 4)] * 4 + [("cfgpp", 1)], pp_backend.log
    assert pp_backend.launches == 7


def test_two_calls_fresh_solver_and_intermediates(pp_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    fn = wrap("flow", ns, "per_sample", cfg_pp=True)
    s = new.DPM_Solver(fn, ns)
    y1, y2 = s.sample(x_T(), steps=5), s.sample(x_T(), steps=5)
    y3, inter = new.DPM_Solver(fn, ns).sample(x_T(), steps=5, return_intermediate=True)
    assert torch.equal(y1, y2) and torch.equal(y1, y3) and len(inter) == 6 and torch.equal(inter[-1], y1)


def test_correcting_xt_fn_runs_after_each_update(pp_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    seen = []

    def fix(x, t, step):
        seen.append(step)
        return 0.5 * x
    y = new.DPM_Solver(wrap("noise", ns, 0.5, cfg_pp=True), ns, correcting_xt_fn=fix).sample(x_T(), steps=4)
    assert seen == [0, 1, 2, 3, 4] and torch.isfinite(y).all()


# ---- batch sharding ------------------------------------------------------------------------------------------------------

def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dpm_solver_b200 import ops
        import dpm_solver_b200 as new
        ops.set_backend(CFGPPOracle())
        ns = product_schedule("flow")
        x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))[2 * rank:2 * rank + 2]
        fn = wrap("flow", ns, torch.tensor([0.3, 1.0, 0.5, 0.2])[2 * rank:2 * rank + 2], cfg_pp=True)
        y = new.DPM_Solver(fn, ns, plan_broadcast=True).sample(x, steps=5, order=2)
        q.put((rank, y))
    finally:
        dist.destroy_process_group()


def test_batch_sharding(pp_backend):
    """Two gloo ranks of two samples each equal the unsharded run of four; g travels with the broadcast plan."""
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
    ns = product_schedule("flow")
    x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))
    fn = wrap("flow", ns, torch.tensor([0.3, 1.0, 0.5, 0.2]), n=4, cfg_pp=True)
    y = new.DPM_Solver(fn, ns).sample(x, steps=5, order=2)
    assert torch.equal(torch.cat([got[0], got[1]]), y)


# ---- rejections ----------------------------------------------------------------------------------------------------------

def _rejections():
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    uc, c = torch.zeros(B, 1), torch.ones(B, 1)
    base = dict(guidance_type="classifier-free", condition=c, unconditional_condition=uc, guidance_scale=0.5)
    bad_wrap = [
        dict(base, condition=[c, c], guidance_scale=[0.5, 0.3], cfg_pp=True),
        dict(base, guidance_rescale=0.7, cfg_pp=True),
        dict(base, apg_eta=0.0, cfg_pp=True),
        dict(base, cfg_zero_star=True, cfg_pp=True),
        dict(guidance_type="uncond", cfg_pp=True),
        dict(guidance_type="classifier", classifier_fn=lambda *a: None, condition=c, cfg_pp=True),
        dict(base, unconditional_condition=None, cfg_pp=True),
        dict(base, cfg_pp=1),
        dict(base, cfg_pp="yes"),
    ]
    for kw in bad_wrap:
        yield lambda kw=kw: new.model_wrapper(aware, ns, **kw)
    fn = new.model_wrapper(aware, ns, cfg_pp=True, **base)
    yield lambda: new.DPM_Solver(fn, ns, algorithm_type="dpmsolver")
    yield lambda: new.DPM_Solver(fn, ns, correcting_x0_fn="dynamic_thresholding")
    yield lambda: new.DPM_Solver(fn, ns, correcting_x0_fn=lambda x0, t: x0)
    yield lambda: new.DPM_Solver(fn, ns, reference_rounding=True)
    s = new.DPM_Solver(fn, ns)
    yield lambda: s.sample(x_T(), steps=6, order=3)
    for method in ("singlestep", "singlestep_fixed", "adaptive"):
        yield lambda method=method: s.sample(x_T(), steps=6, order=2, method=method)
    yield lambda: s.inverse(x_T(), steps=6, order=3)
    yield lambda: new.UniPC(fn, ns).sample(x_T(), steps=6, order=2)
    t1, t0 = torch.tensor([0.8]), torch.tensor([0.6])
    yield lambda: s.dpm_solver_first_update(x_T(), t1, t0)
    yield lambda: s.singlestep_dpm_solver_second_update(x_T(), t1, t0)
    yield lambda: s.singlestep_dpm_solver_third_update(x_T(), t1, t0)
    yield lambda: s.multistep_dpm_solver_second_update(x_T(), [x_T(1), x_T(2)], [torch.tensor([0.9]), t1], t0)
    yield lambda: s.multistep_dpm_solver_third_update(x_T(), [x_T(1), x_T(2), x_T(3)],
                                                      [torch.tensor([0.95]), torch.tensor([0.9]), t1], t0)
    yield lambda: s.multistep_dpm_solver_update(x_T(), [x_T(1), x_T(2)], [torch.tensor([0.9]), t1], t0, 2)
    yield lambda: s.singlestep_dpm_solver_update(x_T(), t1, t0, 2)
    yield lambda: s.dpm_solver_adaptive(x_T(), 2, 1.0, 1e-3)


def test_rejections_launch_nothing(pp_backend):
    n = 0
    for call in _rejections():
        before = pp_backend.launch_count()
        with pytest.raises(ValueError):
            call()
        assert pp_backend.launch_count() == before
        n += 1
    assert n == 27


def test_c_abi_refuses_other_steps():
    """dpm_step_cfgpp takes LIN1 / multistep DIFF2 data-prediction updates of a CFG pair, nothing else (checked before
    any device access)."""
    import ctypes as C
    from dpm_solver_b200 import _lib
    lib = _lib.lib()
    for kw in (dict(form=0), dict(form=5), dict(c0_on_old=1), dict(n_model=1), dict(predict_x0=0), dict(raw_round=1)):
        d = _lib.StepDesc()
        d.n, d.form, d.n_model, d.predict_x0, d.state_dtype, d.model_dtype = 64, 1, 2, 1, 0, 0
        for k, v in kw.items():
            setattr(d, k, v)
        assert lib.dpm_step_cfgpp(C.byref(d), 0.5, None, None) < 0, kw
