"""Adaptive projected guidance (`model_wrapper(..., apg_eta=...)`) on the CPU: the product's host logic on the numpy
executor (tests/apg_oracle.py) against the fp64 transcription of the paper's formulas, against plain CFG at eta = 1,
and sample() against the UNMODIFIED reference solver driven by an fp64 APG data prediction; momentum reset, the scale-1
bypass and the rejections."""
import itertools

import numpy as np
import pytest
import torch

from apg_oracle import APG64, APGOracle, apg_x0_model, reference_solver, x0_fp64
from cases import make_betas
from oracle import ref_loader

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
B, SHAPE = 2, (2, 3, 6, 6)
W = 4.0
MODEL_TYPES = ["noise", "x_start", "v", "score", "flow", "edm"]
PARAM = {"noise": 0, "x_start": 1, "v": 2, "score": 3, "flow": 4, "edm": 5}


@pytest.fixture()
def apg_backend():
    from dpm_solver_b200 import ops
    be = APGOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def net(x, t, c):
    """A time-independent network whose two halves differ nonlinearly."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x + 0.25 * cc * torch.cos(0.7 * x) - 0.1


def product_schedule(mt):
    import dpm_solver_b200 as new
    if mt == "flow":
        return new.NoiseScheduleFlow(shift=3.0)
    if mt == "edm":
        return new.NoiseScheduleEDM()
    return new.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def reference_schedule(mt):
    if mt == "flow":
        from flow_oracle import reference_schedule as flow
        return flow(3.0)
    if mt == "edm":
        from edm_oracle import reference_schedule as edm
        return edm()
    ref = ref_loader.load("dpm_solver_pytorch")
    return ref.NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))


def wrap(mt, ns, w=W, uc=None, c=None, **apg):
    import dpm_solver_b200 as new
    uc = torch.zeros(B, 1) if uc is None else uc
    c = torch.ones(B, 1) if c is None else c
    return new.model_wrapper(net, ns, model_type=mt, guidance_type="classifier-free", condition=c,
                             unconditional_condition=uc, guidance_scale=w, **apg)


def x_T(seed=0):
    return torch.randn(SHAPE, generator=torch.Generator().manual_seed(seed))


def rel_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


# ---- the guided x0 against the paper's formulas ----------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_guided_x0_vs_fp64_transcription(apg_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    ts = [torch.tensor([0.9]), torch.tensor([0.6]), torch.tensor([0.3])]
    xs = [x_T(k) * (1.0 + 0.3 * k) for k in range(3)]
    worst, clipped = 0.0, 0
    for eta, r, beta in itertools.product((0.0, 0.5, 1.0), (0.0, 1e-2, 1e6), (0.0, -0.5, 0.3)):
        s = new.DPM_Solver(wrap(mt, ns, apg_eta=eta, apg_norm_threshold=r, apg_momentum=beta), ns)
        want_fn = APG64(eta, r, beta)
        with s._apg_scope():          # the evaluations of one run: the momentum carries over
            for x, t in zip(xs, ts):
                got = s.data_prediction_fn(x, t).numpy()
                out_u, out_c = net(torch.cat([x, x]), None, torch.cat([torch.zeros(B, 1), torch.ones(B, 1)])).chunk(2)
                al, sg = float(ns.marginal_alpha(t)), float(ns.marginal_std(t))
                sd = getattr(ns, "sigma_data", None)
                c = x0_fp64(PARAM[mt], out_c.numpy(), x.numpy(), al, sg, sd)
                u = x0_fp64(PARAM[mt], out_u.numpy(), x.numpy(), al, sg, sd)
                diff = c - u if want_fn.running is None or beta == 0 else (c - u) + beta * want_fn.running
                clipped += r == 1e-2 and np.sqrt((diff.reshape(B, -1) ** 2).sum(1)).min() > r
                want = want_fn(c, u, W)
                worst = max(worst, rel_err(got, want))
    assert clipped > 0
    assert worst <= 2e-5, worst


@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
def test_eta_one_is_plain_cfg(apg_backend, mt, algo):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    kw = dict(steps=6, order=2, method="multistep")
    y_apg = new.DPM_Solver(wrap(mt, ns, apg_eta=1.0), ns, algorithm_type=algo).sample(x_T(), **kw)
    y_cfg = new.DPM_Solver(wrap(mt, ns), ns, algorithm_type=algo).sample(x_T(), **kw)
    # (for dpmsolver, APG's noise is the guided x0 taken back through (x - alpha*x0)/sigma, where plain CFG combines the
    # noise directly: one more rounding, divided by sigma near the end of the run; measured at most 3.8e-5)
    assert rel_err(y_apg, y_cfg) <= (1e-5 if algo == "dpmsolver++" else 1e-4)


# ---- sample() against the reference ----------------------------------------------------------------------------------

METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2),
           ("singlestep", 3), ("adaptive", 2), ("unipc", 2)]
CONFIGS = [(0.0, 0.0, 0.0, False), (0.3, 2.0, -0.5, False), (0.0, 0.0, 0.3, True)]   # (eta, r, beta, thresholding)


@needs_ref
@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("method,order", METHODS)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
def test_sample_matches_reference(apg_backend, mt, method, order, algo, cfg, capsys):
    import dpm_solver_b200 as new
    eta, r, beta, thr = CONFIGS[cfg]
    if method == "adaptive" and beta != 0:
        pytest.skip("momentum is refused with the adaptive solver (test_rejections_launch_nothing)")
    if thr and algo == "dpmsolver":
        pytest.skip("thresholding acts on the data prediction")
    ns, rns = product_schedule(mt), reference_schedule(mt)
    fn = wrap(mt, ns, apg_eta=eta, apg_norm_threshold=r, apg_momentum=beta)
    tin = getattr(rns, "input_time", None)
    if tin is None:
        tin = lambda t: (t - 1. / rns.total_N) * 1000.
    x0_fn = apg_x0_model(net, rns, PARAM[mt], torch.zeros(B, 1), torch.ones(B, 1), W, eta, r, beta, tin)
    rs = reference_solver(rns, x0_fn, algo, thresholding=thr)
    kw = dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
    if method == "unipc":
        # UniP-2 bh2 without the corrector is DPM-Solver(++)(2M)
        y = new.UniPC(fn, ns, variant="bh2", **kw).sample(x_T(), steps=6, order=2, use_corrector=False)
        yr = rs.sample(x_T(), steps=6, order=2, method="multistep")
    else:
        skw = dict(steps=6, order=order, method=method)
        if method == "adaptive":
            skw = dict(order=order, method=method, atol=0.05, rtol=0.1)
        y = new.DPM_Solver(fn, ns, **kw).sample(x_T(), **skw)
        yr = rs.sample(x_T(), **skw)
    capsys.readouterr()
    # the reference reads an x0 formed in fp64 and rounded once, the product forms it in fp32 op by op; measured at most
    # 4.0e-5 (dpmsolver's x0 -> eps round trip divides by sigma; the adaptive runs amplify), 1e-5 for most cases
    assert rel_err(y, yr) <= 1e-4, rel_err(y, yr)


def test_unipc_launches(apg_backend):
    """UniPC: per evaluation the words pass, one launch that writes the buffered value and a UniPC launch that reads it
    (no network output)."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    y = new.UniPC(wrap("noise", ns, apg_eta=0.2, apg_momentum=-0.5), ns).sample(x_T(), steps=5, order=2)
    assert sum(e[0] == "apg_words" for e in apg_backend.log) == 5
    assert sum(1 for e in apg_backend.log if e[0] == 0 and e[1] == 2) == 5     # FORM_NONE launches on the CFG pair
    assert sum(1 for e in apg_backend.log if e[0] == "unipc" and e[1] == 0) == 4
    assert np.isfinite(y.numpy()).all()


# ---- momentum, bypass, rejections ------------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_two_sample_calls_are_bit_identical(apg_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    s = new.DPM_Solver(wrap(mt, ns, apg_eta=0.0, apg_norm_threshold=2.0, apg_momentum=-0.5), ns)
    y1 = s.sample(x_T(), steps=5, order=2)
    y2 = s.sample(x_T(), steps=5, order=2)
    assert torch.equal(y1, y2)
    u = new.UniPC(wrap(mt, ns, apg_eta=0.0, apg_momentum=0.3), ns)
    assert torch.equal(u.sample(x_T(), steps=5, order=2), u.sample(x_T(), steps=5, order=2))
    # momentum really acts: a run without it differs
    y0 = new.DPM_Solver(wrap(mt, ns, apg_eta=0.0, apg_norm_threshold=2.0), ns).sample(x_T(), steps=5, order=2)
    assert not torch.equal(y0, y1)


@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_scale_one_bypass(apg_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    kw = dict(steps=5, order=2)
    # a scalar scale of 1: one network half, no APG launch, the plain run's launches and result
    apg_backend.log.clear()
    y1 = new.DPM_Solver(wrap(mt, ns, w=1.0, apg_eta=0.0, apg_momentum=-0.5), ns).sample(x_T(), **kw)
    log_apg = list(apg_backend.log)
    apg_backend.log.clear()
    y0 = new.DPM_Solver(wrap(mt, ns, w=1.0), ns).sample(x_T(), **kw)
    assert log_apg == apg_backend.log and torch.equal(y0, y1)
    assert all(e[0] != "apg_words" for e in log_apg)
    # a per-sample scale of 1: that row is c, whatever the other rows and the momentum
    yb = new.DPM_Solver(wrap(mt, ns, w=torch.tensor([1.0, 5.0]), apg_eta=0.0, apg_momentum=-0.5), ns).sample(
        x_T(), **kw)
    assert torch.equal(yb[:1], y0[:1])
    assert not torch.equal(yb[1:], y0[1:])


def test_direct_model_fn_call(apg_backend):
    """model_fn(x, t) returns the guided noise: the guided x0 through the x_start conversion."""
    import dpm_solver_b200 as new
    for mt in MODEL_TYPES:
        ns = product_schedule(mt)
        fn = wrap(mt, ns, apg_eta=0.5, apg_norm_threshold=3.0)
        x, t = x_T(3), torch.full((B,), 0.5)
        eps = fn(x, t).numpy()
        s = new.DPM_Solver(fn, ns)
        x0 = s.data_prediction_fn(x, t[:1]).numpy()
        al, sg = np.float32(ns.marginal_alpha(t[:1])), np.float32(ns.marginal_std(t[:1]))
        assert np.array_equal(eps, ((x.numpy() - al * x0) / sg).astype(np.float32))


def _rejections():
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    uc, c = torch.zeros(B, 1), torch.ones(B, 1)
    base = dict(guidance_type="classifier-free", condition=c, unconditional_condition=uc, guidance_scale=W)
    bad_wrap = [
        dict(base, condition=[c, c], guidance_scale=[2.0, 3.0], apg_eta=0.0),
        dict(base, guidance_rescale=0.7, apg_eta=0.0),
        dict(guidance_type="uncond", apg_eta=0.0),
        dict(base, unconditional_condition=None, apg_eta=0.0),
        dict(base, apg_eta=float("nan")),
        dict(base, apg_eta=0.0, apg_momentum=float("inf")),
        dict(base, apg_eta=0.0, apg_norm_threshold=-1.0),
        dict(base, apg_eta=0.0, apg_norm_threshold=float("inf")),
        dict(base, apg_momentum=0.5),
    ]
    for kw in bad_wrap:
        yield lambda kw=kw: new.model_wrapper(net, ns, **kw)
    fn = new.model_wrapper(net, ns, apg_eta=0.0, **base)
    yield lambda: new.DPM_Solver(fn, ns, reference_rounding=True)
    fm = new.model_wrapper(net, ns, apg_eta=0.0, apg_momentum=-0.5, **base)
    yield lambda: new.DPM_Solver(fm, ns).sample(x_T(), order=2, method="adaptive")
    yield lambda: new.DPM_Solver(fm, ns).inverse(x_T(), order=2, method="adaptive")


def test_rejections_launch_nothing(apg_backend):
    n = 0
    for call in _rejections():
        before = apg_backend.launch_count()
        with pytest.raises(ValueError):
            call()
        assert apg_backend.launch_count() == before
        n += 1
    assert n == 12
