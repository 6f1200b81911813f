"""Flow-matching sampling (`NoiseScheduleFlow`, `model_wrapper(..., model_type="flow")`) on the CPU: the schedule's
scalars against fp64, and the product's host logic on the numpy executor against the UNMODIFIED reference solver driven
on the flow schedule (tests/flow_oracle.py), bit for bit."""
import itertools
import math
import random
from unittest import mock

import numpy as np
import pytest
import torch

from cases import exact_net, seeded
from oracle import ref_loader

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
SHIFTS = [1.0, 3.0, 1.15]
B, SHAPE = 3, (3, 2, 4, 4)


def schedule(shift, **kw):
    from dpm_solver_b200 import NoiseScheduleFlow
    return NoiseScheduleFlow(shift=shift, **kw)


def ulps(a, b64):
    """|a - b| in units of the fp32 spacing at b."""
    b32 = b64.astype(np.float32)
    sp = np.spacing(np.abs(b32)).astype(np.float64)
    return np.abs(a.astype(np.float64) - b64) / np.maximum(sp, 1e-300)


# ---- 1. the schedule ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shift", SHIFTS)
def test_schedule_scalars_match_fp64(shift):
    ns = schedule(shift)
    t = torch.linspace(1e-3, ns.T, 4001)
    t64 = t.double().numpy()
    s32, m1 = np.float64(np.float32(shift)), np.float64(np.float32(shift - 1.))
    sig = s32 * t64 / (1. + m1 * t64)
    assert ulps(ns.marginal_std(t).numpy(), sig).max() <= 3       # four rounded ops
    # alpha, log alpha and lambda inherit the rounding of sigma: compare with the fp64 function of the fp32 inputs
    assert ulps(ns.marginal_alpha(t).numpy(), 1. - ns.marginal_std(t).double().numpy()).max() <= 0.5
    a32, g32 = ns.marginal_alpha(t).double().numpy(), ns.marginal_std(t).double().numpy()
    assert ulps(ns.marginal_log_mean_coeff(t).numpy(), np.log(a32)).max() <= 2
    lam = ns.marginal_lambda(t).numpy()
    assert np.abs(lam - (np.log(a32) - np.log(g32))).max() <= 4 * np.spacing(np.float32(8.))
    la, sg, lm, al = ns.marginals(t)
    for got, want in ((la, ns.marginal_log_mean_coeff(t)), (sg, ns.marginal_std(t)), (lm, ns.marginal_lambda(t)),
                      (al, ns.marginal_alpha(t))):
        assert torch.equal(got, want)


@pytest.mark.parametrize("shift", SHIFTS)
def test_inverse_lambda_round_trip(shift):
    ns = schedule(shift)
    t = torch.linspace(1e-3, ns.T, 2001)
    back = ns.inverse_lambda(ns.marginal_lambda(t))
    # d t / d lambda = sigma*alpha*(...): an ulp of lambda (<= 2^-21 at |lambda| < 8) moves t by less than 1e-6
    assert (back - t).abs().max() <= 4e-6


def test_shift_one_is_the_identity_and_T():
    ns = schedule(1.0)
    t = torch.rand(10000, generator=torch.Generator().manual_seed(0))
    assert torch.equal(ns.marginal_std(t), t)
    assert torch.equal(ns.marginal_alpha(t), 1. - t)
    assert ns.schedule == "flow" and ns.T == 1. - 1. / 1000 and ns.total_N == 1000
    assert schedule(3.0, total_N=50).T == 1. - 1. / 50
    assert math.isfinite(float(ns.marginal_lambda(torch.tensor([ns.T]))))
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError):
            schedule(bad)


@pytest.mark.parametrize("time_scale", [1000.0, 1.0])
def test_model_input_time(time_scale):
    import dpm_solver_b200 as new
    ns = schedule(3.0, time_scale=time_scale)
    seen = []
    fn = new.model_wrapper(lambda x, t: seen.append(t.clone()) or x, ns, model_type="flow")
    t = torch.tensor([0.25, 0.5, 0.75])
    assert torch.equal(fn.get_model_input_time(t), time_scale * ns.marginal_std(t))
    assert torch.equal(fn.get_model_input_time(t), ns.model_input_time(t))


def test_vp_marginals_unchanged():
    """plan.Marginals on a VP schedule: the reference's expressions, and alpha_e is alpha itself."""
    from dpm_solver_b200 import NoiseScheduleVP, plan
    ns = NoiseScheduleVP("linear")
    t = torch.linspace(1e-3, 1., 101)
    m = plan.Marginals(ns, t)
    assert torch.equal(m.alpha, ns.marginal_alpha(t)) and m.alpha_e is m.alpha
    assert torch.equal(m.sigma, ns.marginal_std(t)) and torch.equal(m.lam, ns.marginal_lambda(t))


# ---- 3. rejections -----------------------------------------------------------------------------------------------------

def test_rejections_raise_before_any_launch():
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops

    class NoLaunch:
        def __getattr__(self, name):
            raise AssertionError("the executor was reached: " + name)

    old = ops._backend
    ops.set_backend(NoLaunch())
    try:
        flow, vp = schedule(3.0), new.NoiseScheduleVP("linear")
        net = lambda x, t: x
        with pytest.raises(ValueError, match="NoiseScheduleFlow"):
            new.model_wrapper(net, vp, model_type="flow")
        for mt in ("v", "score"):
            with pytest.raises(ValueError, match="variance-preserving"):
                new.model_wrapper(net, flow, model_type=mt)
        with pytest.raises(ValueError, match="classifier guidance"):
            new.model_wrapper(net, flow, model_type="flow", guidance_type="classifier", classifier_fn=net)
        for mt in ("flow", "noise", "x_start"):
            fn = new.model_wrapper(net, flow, model_type=mt)
            with pytest.raises(ValueError, match="reference_rounding"):
                new.DPM_Solver(fn, flow, reference_rounding=True)
            new.DPM_Solver(fn, flow)
    finally:
        ops.set_backend(old)


# ---- 2. the unmodified reference solver as the oracle -----------------------------------------------------------------

def flow_net(calls=None):
    """Exact IEEE multiplies and adds; the conditional blocks differ in scale and offset."""
    def net(x, t, c=None):
        if calls is not None:
            calls.append((tuple(x.shape), t.tolist()))
        out = exact_net(x.float(), t)
        if c is not None:
            out = out * (1. + 0.3 * c.reshape(-1, 1, 1, 1)) + 0.05 * c.reshape(-1, 1, 1, 1)
        return out
    return net


GUIDANCE = {
    "none": None,
    "scalar": dict(kind="scalar", scales=3.5, K=1),
    "per_sample": dict(kind="per_sample", scales=[7.5, 1.0, -2.0], K=1),
    "multi2": dict(kind="multi", scales=[7.5, -2.0], K=2),
    "multi3": dict(kind="multi", scales=[4.0, 0.0, -1.5], K=3),
}


def make_pair(shift, algo, thr, guidance, phi=0.0, time_scale=1000.0):
    """(reference solver, product solver, reference calls, product calls)."""
    import dpm_solver_b200 as new
    import flow_oracle as F
    rns, pns = F.reference_schedule(shift, time_scale), schedule(shift, time_scale=time_scale)
    rc, pc = [], []
    g = GUIDANCE[guidance]
    uc = torch.zeros(B, 1)
    if g is None:
        rs = F.reference_solver(flow_net(), rns, algo, thr, calls=rc)
        pfn = new.model_wrapper(flow_net(pc), pns, model_type="flow")
    else:
        conds = [torch.full((B, 1), float(k + 1)) for k in range(g["K"])]
        rs = F.reference_solver(flow_net(), rns, algo, thr, calls=rc, phi=phi,
                                guidance=dict(uc=uc, conds=conds, scales=g["scales"], kind=g["kind"]))
        pfn = new.model_wrapper(flow_net(pc), pns, model_type="flow", guidance_type="classifier-free",
                                condition=conds if g["kind"] == "multi" else conds[0], unconditional_condition=uc,
                                guidance_scale=g["scales"], guidance_rescale=phi)
    ps = new.DPM_Solver(pfn, pns, algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
    return rs, ps, rc, pc


@pytest.fixture()
def flow_backend():
    from dpm_solver_b200 import ops
    import flow_oracle as F
    be = F.FlowOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2), ("singlestep", 3),
           ("singlestep_fixed", 2), ("singlestep_fixed", 3)]
SKIPS = ["time_uniform", "logSNR", "time_quadratic"]


def sweep():
    """A seeded sweep of algorithm x method x order x skip type x shift x guidance x thresholding: the full product of
    algorithm, method and guidance, the rest drawn."""
    rng = random.Random(20240)
    out = []
    for algo, (method, order), guidance in itertools.product(("dpmsolver++", "dpmsolver"), METHODS, GUIDANCE):
        thr = algo == "dpmsolver++" and rng.random() < 0.5
        out.append((algo, method, order, rng.choice(SKIPS), rng.choice(SHIFTS), guidance, thr,
                    rng.choice(["dpmsolver", "taylor"]), rng.random() < 0.3))
    return out


@needs_ref
@pytest.mark.parametrize("algo,method,order,skip,shift,guidance,thr,solver_type,d2z", sweep())
def test_sample_matches_reference_solver(flow_backend, algo, method, order, skip, shift, guidance, thr, solver_type, d2z):
    rs, ps, rc, pc = make_pair(shift, algo, thr, guidance)
    x = seeded(SHAPE, 11)
    kw = dict(steps=7, order=order, method=method, skip_type=skip, solver_type=solver_type, denoise_to_zero=d2z,
              return_intermediate=True)
    yr, ir = rs.sample(x.clone(), **kw)
    yp, ip = ps.sample(x.clone(), **kw)
    assert pc == rc                                  # the same (x.shape, t_input) network calls, in the same order
    assert len(ip) == len(ir)
    for a, b in zip(ip, ir):
        np.testing.assert_array_equal(a.numpy(), b.numpy())
    np.testing.assert_array_equal(yp.numpy(), yr.numpy())
    assert yp.isfinite().all()


@needs_ref
@pytest.mark.parametrize("algo,thr", [("dpmsolver++", False), ("dpmsolver++", True), ("dpmsolver", False)])
@pytest.mark.parametrize("method,order", [("multistep", 2), ("singlestep", 3)])
def test_guidance_rescale_matches_reference_solver(flow_backend, algo, thr, method, order):
    """combine and rescale the raw velocities, then convert (the ratio in fp64 on both sides)."""
    rs, ps, rc, pc = make_pair(3.0, algo, thr, "scalar", phi=0.7)
    x = seeded(SHAPE, 5)
    kw = dict(steps=6, order=order, method=method)
    yr, yp = rs.sample(x.clone(), **kw), ps.sample(x.clone(), **kw)
    assert pc == rc and ("ratio", 2) in flow_backend.log
    np.testing.assert_array_equal(yp.numpy(), yr.numpy())


@needs_ref
@pytest.mark.parametrize("algo", ["dpmsolver++", "dpmsolver"])
@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("shift", [1.0, 3.0])
def test_adaptive_matches_reference_solver(flow_backend, algo, order, shift):
    rs, ps, rc, pc = make_pair(shift, algo, False, "scalar")
    x = seeded(SHAPE, 7)
    kw = dict(order=order, method="adaptive", atol=0.05, rtol=0.1)
    nfe = []
    for s in (rs, ps):
        with mock.patch("builtins.print") as pr:
            y = s.sample(x.clone(), **kw)
            nfe.append((pr.call_args[0][-1], y))
    assert nfe[0][0] == nfe[1][0] and len(pc) == len(rc)
    yr, yp = nfe[0][1].numpy(), nfe[1][1].numpy()
    # the error estimate is a mean whose summation order differs from torch's (DESIGN.md section 2)
    assert np.abs(yp.astype(np.float64) - yr).max() / np.abs(yr).max() <= 1e-5


@needs_ref
@pytest.mark.parametrize("model_type", ["noise", "x_start"])
def test_noise_and_x_start_networks_on_the_flow_schedule(flow_backend, model_type):
    """The generic conversions need no VP identity: the reference's own model_wrapper on the flow schedule."""
    import dpm_solver_b200 as new
    import flow_oracle as F
    ref = ref_loader.load("dpm_solver_pytorch")
    rns, pns = F.reference_schedule(3.0), schedule(3.0)
    rns.schedule = "linear"          # the reference's wrapper then hands the network t itself: give it what ours gets
    rfn = ref.model_wrapper(lambda x, t: exact_net(x, rns.input_time(t)), rns, model_type=model_type)
    pfn = new.model_wrapper(exact_net, pns, model_type=model_type)
    x = seeded(SHAPE, 3)
    for algo in ("dpmsolver++", "dpmsolver"):
        yr = ref.DPM_Solver(rfn, rns, algorithm_type=algo).sample(x.clone(), steps=6, order=2, t_start=rns.T, t_end=1. / rns.total_N)
        yp = new.DPM_Solver(pfn, pns, algorithm_type=algo).sample(x.clone(), steps=6, order=2)
        np.testing.assert_array_equal(yp.numpy(), yr.numpy())


@needs_ref
def test_model_fn_direct_call(flow_backend):
    """WrappedModel.__call__ returns eps = x + alpha_t*v, with one time label for the batch and one per sample."""
    rs, ps, _, _ = make_pair(3.0, "dpmsolver", False, "scalar")
    x = seeded(SHAPE, 3)
    for t in (torch.full((B,), 0.6), torch.tensor([0.9, 0.5, 0.2])):
        np.testing.assert_array_equal(ps._wrapped(x, t).numpy(), rs.model(x, t).numpy())


@needs_ref
def test_add_noise_and_inverse(flow_backend):
    rs, ps, _, _ = make_pair(1.15, "dpmsolver++", False, "none")
    x, noise = seeded(SHAPE, 1), seeded((2,) + SHAPE, 2)
    t = torch.tensor([0.3, 0.8])
    np.testing.assert_array_equal(ps.add_noise(x, t, noise=noise).numpy(), rs.add_noise(x, t, noise=noise).numpy())
    kw = dict(steps=5, order=2)
    np.testing.assert_array_equal(ps.inverse(x.clone(), **kw).numpy(), rs.inverse(x.clone(), **kw).numpy())
