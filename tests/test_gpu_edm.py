"""The EDM path on the device: DPM_PARAM_EDM launches of every kind against the numpy executor (tests/edm_oracle.py) bit
for bit -- plain, rescaled, per-sample and multi-condition steps on every dispatch path, dpm_step_unipc, the quantile,
the five dtype pairs, tails, unaligned views, channels_last, IEEE-edge operands, launches across many CTAs and every
tuning, one launch beyond 2^31 elements -- seeded sample() and UniPC.sample() configurations against the executor
(first call, second call, fresh solver, graph replay), fp32 runs against the unmodified reference solver, and the
bf16-state distance to the fp64 transcription."""
import random

import numpy as np
import pytest
import torch

from dpm_solver_b200._lib import FORM_LIN1, PARAM_EDM
from dpm_solver_b200.ops import StepArgs
from edm_oracle import EDMOracle
from oracle import ref_loader
from step_edges import assert_bits_equal

pytestmark = pytest.mark.gpu
f32 = np.float32
BF16, F16 = torch.bfloat16, torch.float16


def _edm(a, rng):
    """An EDM launch from a flow one: the words are launch constants (eps words have a negative second word)."""
    a.param = PARAM_EDM
    if not a.predict_x0 and rng.random() < 0.7:
        a.sigma_e = -a.sigma_e
    return a


# ---- launches ----------------------------------------------------------------------------------------------------------

def test_edm_launches_match_the_executor(cuda_backend):
    """Every form x dtype pair x guidance family (one output, CFG, rescale, per-sample, 2 and 4 conditions) x solver
    space on each dispatch path (direct, TMA ring, tail, unaligned view, ragged samples, device coefficients,
    channels_last), IEEE edges in the network outputs, bit for bit."""
    from test_gpu_flow import FAMILIES, PATHS, build_case, case_specs, to_device
    seen = set()
    for spec in case_specs():
        a, _ = build_case(spec)
        a = _edm(a, np.random.default_rng(spec["seed"] + 7))
        d = to_device(a, spec["path"], np.random.default_rng(spec["seed"] + 1))
        cuda_backend.set_tuning(1 if spec["path"] == "tma" else 2, 0, 0)
        try:
            gm, go = cuda_backend.step(d)
        finally:
            cuda_backend.set_tuning(2, 0, 0)
        with np.errstate(all="ignore"):
            wm, wo = EDMOracle().step(a)
        for g, w, name in ((gm, wm, "m_out"), (go, wo, "out")):
            assert (g is None) == (w is None), (name, spec)
            if g is not None:
                assert_bits_equal(g, w, "%s of %s thr=%s" % (name, spec, a.thr))
        seen.add((spec["fam"], spec["path"]))
    assert len(seen) == len(FAMILIES) * len(PATHS) - 4, seen


def test_dynamic_threshold_of_edm_launches_matches_the_executor(cuda_backend):
    """dpm_dynamic_threshold on EDM x0 (no divisor: the keys are the converted values), packet and element paths."""
    from test_gpu_flow import build_case, case_specs, to_device
    n = 0
    for spec in case_specs()[::5]:
        if not spec["px0"] or spec["fam"] not in ("plain1", "plain2"):
            continue
        a, _ = build_case(dict(spec, path="direct" if spec["path"] in ("tma", "dev_coef") else spec["path"]))
        a = _edm(a, np.random.default_rng(spec["seed"]))
        for nm in ("e_cond", "e_uncond"):           # finite operands: a NaN makes every threshold NaN
            t = getattr(a, nm)
            if t is not None:
                setattr(a, nm, torch.nan_to_num(t.float(), nan=0.5, posinf=3.0, neginf=-3.0).clamp(-1e4, 1e4).to(t.dtype))
        a.thr = None
        d = to_device(a, "direct", np.random.default_rng(0))
        got = cuda_backend.dynamic_threshold(d, 0.995, 1.0)
        with np.errstate(all="ignore"):
            want = EDMOracle().dynamic_threshold(a, 0.995, 1.0)
        assert_bits_equal(got, want, str(spec))
        n += 1
    assert n >= 20, n


@pytest.mark.parametrize("tuning", [(2, 0, 0), (0, 128, 0), (0, 64, 2), (2, 256, 1)])
def test_unipc_launches_match_the_executor(cuda_backend, tuning):
    """dpm_step_unipc with DPM_PARAM_EDM: every (pc, pp) x network-output count, dtype pairs, thresholds, layouts
    (contiguous, unaligned view, channels_last), IEEE edges."""
    from test_gpu_unipc import build_args, launch_case, same
    rng = random.Random(5000 + tuning[1] + tuning[2])
    ora = EDMOracle()
    cuda_backend.set_tuning(*tuning)
    try:
        seen = set()
        for k in range(150):
            c = launch_case(rng, None)
            c["param"] = PARAM_EDM
            seen.add((c["pc"], c["pp"], c["ne"]))
            a_d = build_args(c, "cuda", torch.Generator().manual_seed(k))
            a_h = build_args(c, "cpu", torch.Generator().manual_seed(k))
            if c["thr"]:
                a_d.thr = a_h.thr.cuda()
            m_d, o_d = cuda_backend.step(a_d)
            m_h, o_h = ora.step(a_h)
            if c["ne"] > 0:
                assert same(m_d, m_h), c
            if c["pp"] > 0:
                assert same(o_d, o_h), c
                if c["out2"]:
                    assert same(a_d.out2, o_h), c
            if c["out_c"]:
                assert same(a_d.out_c, a_h.out_c), c
        torch.cuda.synchronize()
        assert len(seen) >= 30
    finally:
        cuda_backend.set_tuning(2, 0, 0)


def test_edm_launches_across_ctas_and_tunings(cuda_backend):
    """About 3.5 passes of the largest capped grid: the direct, TMA and multi-condition kernels and dpm_step_unipc
    (FAST and generic, both threshold layouts), the default tuning against the executor, every other tuning equal to
    it."""
    import test_gpu_unipc_tiles as T
    per8, per_odd = T.per_sample_sizes()
    for c in T.flow_cases():
        host = T.flow_args(c, per8, per_odd)
        host.param, host.alpha_e, host.sigma_e = PARAM_EDM, 0.392, 0.981 if c["px0"] else -0.196
        with np.errstate(all="ignore"):
            wm, wo = EDMOracle().step(host)
        d = T._to(host, "cuda")
        variant = 1 if c["path"] == "tma" else 2
        m0, o0 = (t.clone() for t in T._launch_flow(cuda_backend, d, (variant, 0, 0)))
        assert_bits_equal(m0, wm, "m_out %s" % c)
        assert_bits_equal(o0, wo, "out %s" % c)
        del wm, wo, host
        for threads, ctas in T.TUNINGS:
            m, o = T._launch_flow(cuda_backend, d, (variant, threads, ctas))
            assert T._same(m, m0) and T._same(o, o0), (threads, ctas, c)
            del m, o
        del d, m0, o0
    for c in T.unipc_cases()[::3]:
        if not c["ne"]:
            continue
        c = dict(c, param=PARAM_EDM)
        host = T.unipc_args(c, per8 if c["mult8"] else per_odd)
        host.out_c = torch.empty_like(host.x)
        with np.errstate(all="ignore"):
            wm, wo = EDMOracle().step(host)
        d = T._to(host, "cuda")
        m0, o0, o20, oc0 = T._launch(cuda_backend, d)
        assert_bits_equal(m0, wm, "m_out %s" % c)
        if c["pp"]:
            assert_bits_equal(o0, wo, "out %s" % c)
        assert_bits_equal(oc0, host.out_c, "out_c %s" % c)
        del wm, wo, host
        for threads, ctas in T.TUNINGS[::3]:
            got = T._launch(cuda_backend, d, (2, threads, ctas))
            for g, w in zip(got, (m0, o0, o20, oc0)):
                assert (g is None) == (w is None) and (g is None or T._same(g, w)), (threads, ctas, c)
        del d, m0, o0, o20, oc0


def test_one_launch_beyond_2_31_elements(cuda_backend):
    """bf16 LIN1 step of an EDM network over 2^31 + 1003 elements against separate torch CUDA ops: x0 = a*x + b*F
    (rounded to bf16 as the buffered value), x_t = a'*x + c0*x0."""
    n = (1 << 31) + 1003
    g = torch.Generator(device="cuda").manual_seed(3)
    x, ec = (torch.randn(n, device="cuda", generator=g).to(BF16) for _ in range(2))
    A, S, a, c0 = 0.098, 0.4905, 0.9375, -0.3125
    m, o = cuda_backend.step(StepArgs(form=FORM_LIN1, n_model=1, x=x, e_cond=ec, param=PARAM_EDM, predict_x0=True,
                                      alpha_e=A, sigma_e=S, a=a, c0=c0, want_m_out=True, state_dtype=BF16))
    step = 1 << 28
    for s0 in range(0, n, step):
        sl = slice(s0, min(n, s0 + step))
        T = (float(f32(A)) * x[sl].float() + float(f32(S)) * ec[sl].float()).to(BF16)
        want = (a * x[sl].float() + c0 * T.float()).to(BF16)
        assert torch.equal(m[sl], T) and torch.equal(o[sl], want), s0


# ---- sample() ----------------------------------------------------------------------------------------------------------

def edm_net(x, t, c=None):
    """Exact IEEE multiplies and adds of the input and c_noise: the same bits on CPU and CUDA."""
    out = 0.1 * x + ((t * 0.25) - 0.02).reshape(-1, *([1] * (x.dim() - 1)))
    return out if c is None else out * (1. + 0.3 * c.reshape(-1, *([1] * (x.dim() - 1)))) + 0.05 * c.reshape(
        -1, *([1] * (x.dim() - 1)))


def draw(rng):
    unipc = rng.random() < 0.35
    steps = rng.randint(2, 12)
    order = rng.randint(1, min(3, steps))
    guidance = rng.choice(["none", "scalar", "rescale"] if unipc else
                          ["none", "scalar", "scalar", "rescale", "per_sample", "multi2"])
    method = "multistep" if unipc else rng.choice(["multistep", "multistep", "singlestep", "singlestep_fixed"])
    if method == "singlestep_fixed":
        order = rng.randint(1, 3)
    if unipc and guidance == "rescale":
        guidance = "scalar"
    return dict(unipc=unipc, steps=steps, order=order, method=method, guidance=guidance,
                alg=rng.choice(["dpmsolver++", "dpmsolver++", "dpmsolver"]), thr=rng.random() < 0.3,
                skip=rng.choice(["time_uniform", "logSNR", "time_quadratic", "karras", "karras"]),
                sd=rng.choice([None, None, BF16, F16]), d2z=rng.random() < 0.3, variant=rng.choice(["bh1", "bh2"]),
                corr=rng.random() < 0.8, shape=rng.choice([(4, 16, 16), (3, 8, 8), (4, 64, 64), (1, 7, 5)]),
                B=rng.choice([1, 2, 3]), sched=rng.choice([dict(), dict(sigma_data=1.0), dict(sigma_min=0.03,
                                                                                             sigma_max=14.6)]))


def make(c, dev):
    import dpm_solver_b200 as new
    ns = new.NoiseScheduleEDM(**c["sched"])
    B, g = c["B"], c["guidance"]
    kw = dict(model_type="edm")
    if g != "none":
        uc = torch.zeros(B, device=dev)
        conds = [torch.full((B,), float(k + 1), device=dev) for k in range(2 if g == "multi2" else 1)]
        scales = {"scalar": 3.5, "rescale": 5.0, "per_sample": [7.5, 1.0, -2.0][:B], "multi2": [7.5, -2.0]}[g]
        kw.update(guidance_type="classifier-free", condition=conds if g == "multi2" else conds[0],
                  unconditional_condition=uc, guidance_scale=scales, guidance_rescale=0.7 if g == "rescale" else 0.)
    fn = new.model_wrapper(edm_net, ns, **kw)
    thr = "dynamic_thresholding" if c["thr"] and c["alg"] == "dpmsolver++" else None
    if c["unipc"]:
        return new.UniPC(fn, ns, algorithm_type=c["alg"], variant=c["variant"], state_dtype=c["sd"],
                         correcting_x0_fn=thr)
    return new.DPM_Solver(fn, ns, algorithm_type=c["alg"], state_dtype=c["sd"], correcting_x0_fn=thr)


def kwargs(c):
    kw = dict(steps=c["steps"], order=c["order"], skip_type=c["skip"], denoise_to_zero=c["d2z"])
    if c["unipc"]:
        kw["use_corrector"] = c["corr"]
    else:
        kw["method"] = c["method"]
    return kw


def same(a, b):
    a, b = a.detach().cpu(), b.detach().cpu()
    return a.dtype == b.dtype and a.shape == b.shape and bool(
        ((a.float() == b.float()) | (torch.isnan(a.float()) & torch.isnan(b.float()))).all())


@pytest.mark.parametrize("chunk", range(3))
def test_sample_matches_the_executor(chunk):
    from dpm_solver_b200 import ops
    rng = random.Random(9100 + chunk)
    old = ops._backend
    try:
        for k in range(20):
            c = draw(rng)
            x = torch.randn(c["B"], *c["shape"], generator=torch.Generator().manual_seed(k)) * 1.0
            ops.set_backend(EDMOracle())
            y_h = make(c, "cpu").sample(x.clone(), **kwargs(c))
            ops.set_backend(ops.CudaBackend())
            s = make(c, "cuda")
            xd = x.cuda()
            assert same(s.sample(xd, **kwargs(c)), y_h), c                    # first call
            assert same(s.sample(xd, **kwargs(c)), y_h), c                    # second call (prepared launches)
            assert same(make(c, "cuda").sample(xd, **kwargs(c)), y_h), c      # fresh solver
            if not c["thr"]:          # (the thresholded step allocates its quantile workspace per call)
                g = make(c, "cuda").capture(xd, **kwargs(c))
                assert same(g(xd), y_h), c
            torch.cuda.synchronize()
    finally:
        ops.set_backend(old)


needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")


@needs_ref
@pytest.mark.parametrize("algo,method,order,guidance,thr", [
    ("dpmsolver++", "multistep", 2, "none", False), ("dpmsolver++", "multistep", 3, "scalar", True),
    ("dpmsolver", "singlestep", 3, "scalar", False), ("dpmsolver++", "singlestep_fixed", 2, "multi2", True)])
def test_fp32_matches_the_reference_solver(cuda_backend, algo, method, order, guidance, thr):
    """c2-like latents ([4, 4, 64, 64], fp32), Karras's grid (time_uniform), denoise_to_zero."""
    import dpm_solver_b200 as new
    import edm_oracle as E
    from test_edm import GUIDANCE, edm_net as net_with_calls
    B = 4
    g = GUIDANCE[guidance]
    conds = None if g is None else [torch.full((B, 1), float(k + 1)) for k in range(g["K"])]
    scales = None if g is None else (g["scales"] if g["kind"] != "per_sample" else g["scales"] + [3.5])
    gd = None if g is None else dict(uc=torch.zeros(B, 1), conds=conds, scales=scales, kind=g["kind"])
    rs = E.reference_solver(net_with_calls(), E.reference_schedule(), algo, thr, **({} if gd is None else dict(guidance=gd)))
    x = torch.randn(B, 4, 64, 64, generator=torch.Generator().manual_seed(31)) * 80.
    kw = dict(steps=10, order=order, method=method, denoise_to_zero=True)
    want = rs.sample(x.clone(), **kw)
    pns = new.NoiseScheduleEDM()
    if g is None:
        fn = new.model_wrapper(net_with_calls(), pns, model_type="edm")
    else:
        cd = [c.cuda() for c in conds]
        fn = new.model_wrapper(net_with_calls(), pns, model_type="edm", guidance_type="classifier-free",
                               condition=cd if g["kind"] == "multi" else cd[0],
                               unconditional_condition=torch.zeros(B, 1, device="cuda"), guidance_scale=scales)
    ps = new.DPM_Solver(fn, pns, algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)
    assert_bits_equal(ps.sample(x.cuda(), **kw), want, "first call")
    assert_bits_equal(ps.sample(x.cuda(), **kw), want, "second call")


# ---- bf16 distance -------------------------------------------------------------------------------------------------------

# max |y_N(bf16 state) - y_N(fp64)| / max |y_N(fp64)| on the configuration below, measured on an H100 (DESIGN.md §8.11)
BF16_DISTANCE = 2.33e-2


def test_bf16_state_distance_to_the_fp64_transcription(cuda_backend):
    """c2-like: the default EDM schedule, an EDM network, dpmsolver++, UniPC-2 bh2 with the corrector, 20 steps on
    Karras's grid."""
    import dpm_solver_b200 as new
    from dpm_solver_b200 import plan as P
    from unipc_oracle import unipc_fp64
    ns = new.NoiseScheduleEDM()
    net = lambda y, t: 0.1 * y + ((t * 0.25) - 0.02).reshape(-1, 1, 1, 1)
    x = torch.randn(8, 4, 64, 64, generator=torch.Generator().manual_seed(2))
    y = new.UniPC(new.model_wrapper(net, ns, model_type="edm"), ns, state_dtype=BF16).sample(x.cuda(), steps=20,
                                                                                             order=2)
    s = new.UniPC(new.model_wrapper(net, ns, model_type="edm"), ns)
    ts = s.get_time_steps("time_uniform", ns.T, 1. / ns.total_N, 20, "cpu")
    marg = P.Marginals(ns, ts)
    lam, al, sg, ae = (v.double().numpy() for v in (marg.lam, marg.alpha, marg.sigma, marg.alpha_e))
    tin = ns.model_input_time(ts).double().numpy()
    sd = ns.sigma_data

    def model(yy, i):
        F = 0.1 * yy + (tin[i] * 0.25 - 0.02)
        return sd * sd * ae[i] * yy + sd * sg[i] * F

    y64 = unipc_fp64(model, al, sg, lam, x.double().numpy(), 2)
    d = float(np.abs(y.double().cpu().numpy() - y64).max() / np.abs(y64).max())
    print("bf16 state distance to fp64:", d)
    assert d <= 1.5 * BF16_DISTANCE, d
