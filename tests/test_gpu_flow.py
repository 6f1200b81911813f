"""The flow-matching path on the device: DPM_PARAM_FLOW launches on every dispatch path against the numpy executor
(tests/flow_oracle.py) with IEEE edge operands in the velocities, against two launches of kernels that existed before
(division by 1 is exact), the kernel names torch.profiler reports, dynamic thresholding against torch.quantile, sample()
against the unmodified reference solver driven on the flow schedule, and the device adaptive controller."""
import dataclasses
import os
import subprocess
import sys
from collections import Counter
from unittest import mock

import numpy as np
import pytest
import torch

from cases import seeded
from dpm_solver_b200._lib import FORM_DIFF2, FORM_LIN1, FORM_NONE, FORM_SS3T, PARAM_FLOW, PARAM_NOISE, PARAM_V
from dpm_solver_b200.ops import StepArgs
from flow_oracle import FlowOracle
from oracle import ref_loader
from step_edges import assert_bits_equal, scatter_edges

pytestmark = pytest.mark.gpu
f32 = np.float32
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
PAIRS = [(F32, F32), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32)]      # (model, state)
PATHS = ("direct", "tma", "tail", "unaligned", "ragged", "dev_coef", "cl")
FAMILIES = ("plain1", "plain2", "rs", "pg", "multi2", "multi4")
ORDINARY = [0.9, -0.3, 0.2, 0.1, 1.5, 0.7, 0.4, 0.6, -1.1]
SCALES = [7.5, 1.0, 0.0, -2.0, 3.5]
COEF_NAMES = ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e")
TENSORS = ("x", "xe", "m1", "m2", "e_cond", "e_uncond")


def _pick(rng, seq):
    return seq[int(rng.integers(len(seq)))]


def _offset(t, k):
    buf = torch.empty(t.numel() + k, dtype=t.dtype, device="cuda")
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


def build_case(spec):
    """StepArgs on the host for one seeded flow launch; edge operands go into the velocities."""
    rng = np.random.default_rng(spec["seed"])
    fam, path, form, md, sd, px0 = (spec[k] for k in ("fam", "path", "form", "md", "sd", "px0"))
    B, ps = {"tail": (3, 67), "ragged": (6, 12)}.get(path, (4, 64))
    shape = (B, 4, 4, 4) if path == "cl" else (B, ps)
    n = B * ps
    coef = {k: float(f32(_pick(rng, ORDINARY))) for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3")}
    a = StepArgs(form=form, n_model=1 if fam == "plain1" else 2, param=PARAM_FLOW, predict_x0=px0,
                 c0_on_old=bool(rng.random() < 0.5), alpha_e=float(f32(_pick(rng, [0.4, 1e-3, 0.97]))),
                 sigma_e=float(f32(_pick(rng, [0.6, 0.999, 0.03]))), w4=float(f32(_pick(rng, [0.3, 2.0 ** -20]))),
                 guidance=float(_pick(rng, SCALES)), want_m_out=True, state_dtype=sd, per_sample=ps, **coef)
    streams, dtypes = {}, {}

    def add(name, dt):
        streams[name] = rng.standard_normal(n).astype(f32)
        dtypes[name] = dt
    names = ["e_cond"] + (["e_uncond"] if a.n_model == 2 else [])
    K = int(fam[5:]) if fam.startswith("multi") else 0
    names += ["ec%d" % k for k in range(1, K)]
    for nm in names:
        add(nm, md)
    scatter_edges(streams, dtypes, rng)
    plain = {}
    for nm, on in (("x", form != FORM_NONE), ("xe", True), ("m1", form in (2, 3, 4, 5, 6)), ("m2", form in (3, 5, 6))):
        if on:
            plain[nm] = rng.standard_normal(n).astype(f32)
    if rng.random() < 0.3 and form != FORM_NONE:
        plain.pop("xe")                  # the model was evaluated at x itself
    ten = lambda v, dt: torch.from_numpy(v).to(dt).reshape(shape)
    for nm, v in plain.items():
        setattr(a, nm, ten(v, sd))
    for nm in ("e_cond", "e_uncond"):
        if nm in streams:
            setattr(a, nm, ten(streams[nm], md))
    if K:
        a.e_conds = (a.e_cond,) + tuple(ten(streams["ec%d" % k], md) for k in range(1, K))
        a.scales = tuple(float(_pick(rng, SCALES)) for _ in range(K))
    if fam == "rs" or (fam == "pg" and rng.random() < 0.5):
        a.ratio, a.phi = torch.from_numpy((0.5 + rng.random(B)).astype(f32)), 0.7
    if fam == "pg":
        a.guidance_b = torch.tensor([_pick(rng, SCALES) for _ in range(B)], dtype=F32)
    if px0 and path != "tma" and rng.random() < 0.5:
        a.thr = torch.from_numpy(np.array([_pick(rng, [1.0, 1.3, 0.6, 2.5, 2.0 ** 21]) for _ in range(B)], f32))
    return a, n


def to_device(a, path, rng):
    d = dataclasses.replace(a)
    k = int(rng.integers(1, 9)) if path == "unaligned" else 0
    which = _pick(rng, [t for t in TENSORS if getattr(a, t) is not None]) if k else None

    def dev(t, name=None):
        if t is None:
            return None
        if path == "cl":
            return t.cuda().contiguous(memory_format=torch.channels_last)
        return _offset(t, k) if name == which and k else t.cuda()
    for nm in TENSORS:
        setattr(d, nm, dev(getattr(a, nm), nm))
    for nm in ("thr", "ratio", "guidance_b"):
        setattr(d, nm, None if getattr(a, nm) is None else getattr(a, nm).cuda())
    if a.e_conds is not None:
        d.e_conds = (d.e_cond,) + tuple(dev(e) for e in a.e_conds[1:])
    if path == "dev_coef":
        d.coef_dev = torch.tensor([getattr(a, c) for c in COEF_NAMES] + [0.] * 5, dtype=F32).cuda()
        for c in COEF_NAMES:
            setattr(d, c, 123.0)          # the by-value fields are not read
    return d


def case_specs():
    specs, seed = [], 0
    for fam in FAMILIES:
        for path in PATHS:
            if path == "tma" and fam not in ("plain1", "plain2"):
                continue
            for form in range(7):
                for md, sd in PAIRS:
                    for px0 in (True, False):
                        seed += 1
                        specs.append(dict(fam=fam, path=path, form=form, md=md, sd=sd, px0=px0, seed=70000 + seed))
    return specs


def test_flow_launches_match_the_executor(cuda_backend):
    """Every form x dtype pair x guidance family x solver space on each dispatch path, bit for bit."""
    tally = Counter()
    for spec in case_specs():
        a, n = build_case(spec)
        d = to_device(a, spec["path"], np.random.default_rng(spec["seed"] + 1))
        cuda_backend.set_tuning(1 if spec["path"] == "tma" else 2, 0, 0)
        try:
            gm, go = cuda_backend.step(d)
        finally:
            cuda_backend.set_tuning(2, 0, 0)
        with np.errstate(all="ignore"):
            wm, wo = FlowOracle().step(a)
        for g, w, name in ((gm, wm, "m_out"), (go, wo, "out")):
            assert (g is None) == (w is None), (name, spec)
            if g is not None:
                assert_bits_equal(g, w, "%s of %s thr=%s" % (name, spec, a.thr))
        tally[(spec["fam"], spec["path"])] += 1
    assert len(tally) == len(FAMILIES) * len(PATHS) - 4 * 1, tally


def test_dynamic_threshold_of_edge_launch_inputs_matches_the_executor(cuda_backend):
    """dpm_dynamic_threshold on flow launches (small samples: the cluster kernel, packet and element paths)."""
    for spec in case_specs()[::7]:
        if not spec["px0"] or spec["fam"] not in ("plain1", "plain2"):
            continue
        a, n = build_case(dict(spec, path="direct" if spec["path"] in ("tma", "dev_coef") else spec["path"]))
        for nm in ("e_cond", "e_uncond"):           # finite operands: a NaN makes every threshold NaN
            t = getattr(a, nm)
            if t is not None:
                setattr(a, nm, torch.nan_to_num(t.float(), nan=0.5, posinf=3.0, neginf=-3.0).clamp(-1e4, 1e4).to(t.dtype))
        a.thr = None
        d = to_device(a, "direct", np.random.default_rng(0))
        got = cuda_backend.dynamic_threshold(d, 0.995, 1.0)
        with np.errstate(all="ignore"):
            want = FlowOracle().dynamic_threshold(a, 0.995, 1.0)
        assert_bits_equal(got, want, str(spec))


# ---- an oracle that needs nothing but the device ----------------------------------------------------------------------

def _full(shape, dtype, seed, edges):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(shape, device="cuda", dtype=torch.float32, generator=g)
    if edges:
        pool = torch.tensor([float("nan"), float("inf"), -float("inf"), 0.0, -0.0, 1e-45, 1e-40, 3e38, -3e38, 1e-25, 1e30],
                            device="cuda")
        idx = torch.randint(0, t.numel(), (t.numel() // 50,), device="cuda", generator=g)
        t.view(-1)[idx] = pool[torch.randint(0, pool.numel(), (idx.numel(),), device="cuda", generator=g)]
    return t.to(dtype)


@pytest.mark.parametrize("edges", [False, True])
@pytest.mark.parametrize("shape,px0,cfg", [((4096, 4, 64, 64), True, False), ((2048, 4, 64, 64), False, True)])
def test_flow_launch_equals_existing_kernels_with_unit_divisor(cuda_backend, shape, px0, cfg, edges):
    """dpmsolver++: x0 = x - sigma*v is the NOISE launch's (x - sigma*eps)/alpha with alpha = 1; dpmsolver:
    eps = x + alpha*v is the V launch's alpha*out + sigma*x with sigma = 1. The c2 and c3 shapes in bf16."""
    x, m1 = _full(shape, BF16, 1, False), _full(shape, BF16, 2, False)
    ec = _full(shape, BF16, 3, edges)
    eu = _full(shape, BF16, 4, edges) if cfg else None
    base = dict(form=FORM_DIFF2, n_model=2 if cfg else 1, x=x, m1=m1, e_cond=ec, e_uncond=eu, guidance=7.5,
                predict_x0=px0, a=0.9, c0=-0.3, c1=0.2, w0=1.5, want_m_out=True, state_dtype=BF16)
    fm, fo = cuda_backend.step(StepArgs(param=PARAM_FLOW, alpha_e=0.4, sigma_e=0.6, **base))
    if px0:
        om, oo = cuda_backend.step(StepArgs(param=PARAM_NOISE, alpha_e=1.0, sigma_e=0.6, **base))
    else:
        om, oo = cuda_backend.step(StepArgs(param=PARAM_V, alpha_e=0.4, sigma_e=1.0, **base))
    for got, want in ((fm, om), (fo, oo)):
        same = (got.view(torch.int16) == want.view(torch.int16)) | (got.isnan() & want.isnan())
        assert bool(same.all()), int((~same).sum())


def profile_flow_kernels():
    """One flow launch at the c2 shape per solver space, with and without CFG, inside one profiler session: each must
    be a FAST instantiation of the direct kernel."""
    from dpm_solver_b200 import ops
    from torch.profiler import ProfilerActivity, profile
    be = ops.CudaBackend()
    shape = (4096, 4, 64, 64)
    x, m1, ec = (_full(shape, BF16, s, False) for s in (1, 2, 3))
    cases = [(px0, cfg) for px0 in (True, False) for cfg in (False, True)]
    args = [StepArgs(form=FORM_DIFF2, n_model=2 if cfg else 1, x=x, m1=m1, e_cond=ec, e_uncond=m1 if cfg else None,
                     guidance=7.5, param=PARAM_FLOW, predict_x0=px0, alpha_e=0.4, sigma_e=0.6, a=0.9, c0=-0.3, c1=0.2,
                     w0=1.5, want_m_out=True, state_dtype=BF16) for px0, cfg in cases]
    for a in args:
        be.step(a)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for a in args:
            be.step(a)
        torch.cuda.synchronize()
    ran = [e.name.replace(" ", "") for e in prof.events() if "k_step_" in e.name]
    want = ["k_step_direct<__nv_bfloat16,__nv_bfloat16,%d,%d,true,false,false,false>" % (2 if cfg else 1, FORM_DIFF2)
            for _, cfg in cases]
    assert len(ran) == len(want) and all(w in r for w, r in zip(want, ran)), (want, ran)
    print("%d profiled flow launches ran FAST kernels" % len(ran))


def test_profiler_names_a_fast_kernel():
    """profile_flow_kernels() in a child process of its own: a profiler session opened in this process would add to
    the sessions tests/test_gpu_step_edges.py opens here later, and sessions opened after many others in one process
    were seen to record no kernels."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path[:0] = %r; import test_gpu_flow as t; t.profile_flow_kernels()"
            % [root, os.path.join(root, "tests"), os.path.join(root, "tests", "golden")])
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-4000:], r.stderr[-4000:])
    print(r.stdout.strip().splitlines()[-1])


# ---- dynamic thresholding -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("impl", ["pipeline", "cluster"])
@pytest.mark.parametrize("cfg", [False, True])
def test_flow_thresholds_equal_torch_quantile(cuda_backend, impl, cfg):
    """Both quantile paths on the flow x0 = x - sigma*v (formed here by separate torch ops), ties and the floor included."""
    B, ps, sigma, s = 5, 3 * 64 * 64, 0.6, 3.5
    x, v, u = (seeded((B, ps), k) for k in (1, 2, 3))
    v[1] = (v[1] * 4).round() / 4          # a few distinct values: ties at the order statistics
    x[1] = (x[1] * 4).round() / 4
    x[2], v[2], u[2] = x[2] * 0.01, v[2] * 0.01, u[2] * 0.01    # below the floor max_val = 1
    x0 = x - sigma * v
    if cfg:
        x0u = x - sigma * u
        x0 = x0u + s * (x0 - x0u)
    want = torch.maximum(torch.quantile(x0.abs(), 0.995, dim=1), torch.ones(B))
    a = StepArgs(n_model=2 if cfg else 1, e_cond=v.cuda(), e_uncond=u.cuda() if cfg else None, xe=x.cuda(), guidance=s,
                 param=PARAM_FLOW, predict_x0=True, alpha_e=0.4, sigma_e=sigma, per_sample=ps, state_dtype=F32)
    with mock.patch.dict(os.environ, {"DPM_QUANTILE_IMPL": "c"} if impl == "cluster" else {}):
        got, hdr = cuda_backend.dynamic_threshold(a, 0.995, 1.0, return_stats=True)
    assert_bits_equal(got, want, impl)
    assert float(got[2]) == 1.0
    if impl == "pipeline":
        assert hdr is not None and set(hdr[:, 4].tolist()) <= {1, 2}      # the pipeline finished every sample (bracket or exact fallback)


# ---- sample() -----------------------------------------------------------------------------------------------------------

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no oracle/_ref")
CONFIGS = [("dpmsolver++", "multistep", 2, "none", False), ("dpmsolver++", "multistep", 3, "scalar", True),
           ("dpmsolver", "singlestep", 3, "scalar", False), ("dpmsolver++", "singlestep", 2, "per_sample", True),
           ("dpmsolver", "multistep", 2, "multi2", False), ("dpmsolver++", "singlestep_fixed", 2, "multi3", True)]


def _product(cuda, algo, guidance, thr, state_dtype=None, shift=3.0, shape=(3, 4, 16, 16)):
    import dpm_solver_b200 as new
    from test_flow import GUIDANCE, flow_net
    dev = "cuda" if cuda else "cpu"
    pns, g = new.NoiseScheduleFlow(shift=shift), GUIDANCE[guidance]
    if g is None:
        fn = new.model_wrapper(flow_net(), pns, model_type="flow")
    else:
        conds = [torch.full((shape[0], 1), float(k + 1), device=dev) for k in range(g["K"])]
        fn = new.model_wrapper(flow_net(), pns, model_type="flow", guidance_type="classifier-free",
                               condition=conds if g["kind"] == "multi" else conds[0],
                               unconditional_condition=torch.zeros(shape[0], 1, device=dev), guidance_scale=g["scales"])
    return new.DPM_Solver(fn, pns, algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None,
                          state_dtype=state_dtype)


@needs_ref
@pytest.mark.parametrize("algo,method,order,guidance,thr", CONFIGS)
def test_sample_matches_reference_solver_on_the_device(cuda_backend, algo, method, order, guidance, thr):
    import flow_oracle as F
    from test_flow import GUIDANCE, flow_net
    shape = (3, 4, 16, 16)
    g = GUIDANCE[guidance]
    gd = None if g is None else dict(uc=torch.zeros(3, 1), conds=[torch.full((3, 1), float(k + 1)) for k in range(g["K"])],
                                     scales=g["scales"], kind=g["kind"])
    rs = F.reference_solver(flow_net(), F.reference_schedule(3.0), algo, thr, **({} if gd is None else dict(guidance=gd)))
    x = seeded(shape, 21)
    kw = dict(steps=8, order=order, method=method, denoise_to_zero=True)
    want = rs.sample(x.clone(), **kw)
    ps = _product(True, algo, guidance, thr)
    first = ps.sample(x.cuda(), **kw)
    assert_bits_equal(first, want, "first call")
    assert_bits_equal(ps.sample(x.cuda(), **kw), want, "second call (prepared launches)")
    assert_bits_equal(_product(True, algo, guidance, thr).sample(x.cuda(), **kw), want, "fresh solver")
    if not thr:          # (the thresholded step allocates its quantile workspace per call)
        replay = ps.capture(x.cuda(), **kw)
        assert_bits_equal(replay(x.cuda()), want, "capture() replay")


@pytest.mark.parametrize("algo,method,order,guidance,thr", CONFIGS)
@pytest.mark.parametrize("sd", [BF16, F16])
def test_16_bit_state_matches_the_executor(cuda_backend, algo, method, order, guidance, thr, sd):
    from dpm_solver_b200 import ops
    x = seeded((3, 4, 16, 16), 22)
    kw = dict(steps=8, order=order, method=method)
    got = _product(True, algo, guidance, thr, sd).sample(x.cuda(), **kw)
    ops.set_backend(FlowOracle())
    try:
        want = _product(False, algo, guidance, thr, sd).sample(x.clone(), **kw)
    finally:
        ops.set_backend(cuda_backend)
    assert got.dtype == sd
    assert_bits_equal(got, want, "16-bit state")


def test_channels_last_and_diffedit_helpers(cuda_backend):
    ps = _product(True, "dpmsolver++", "scalar", False)
    x = seeded((3, 4, 16, 16), 23).cuda()
    kw = dict(steps=6, order=2)
    assert_bits_equal(ps.sample(x.contiguous(memory_format=torch.channels_last), **kw), ps.sample(x, **kw), "channels_last")
    t = torch.tensor([0.3, 0.8])
    noise = seeded((2, 3, 4, 16, 16), 24).cuda()
    ns = ps.noise_schedule
    want = torch.stack([float(ns.marginal_alpha(t[i:i + 1])) * x + float(ns.marginal_std(t[i:i + 1])) * noise[i]
                        for i in range(2)])
    assert_bits_equal(ps.add_noise(x, t, noise=noise), want, "add_noise")


# ---- the device adaptive controller -------------------------------------------------------------------------------------
# The controller's contract (csrc/adaptive_ctl.cu): the host's fp32 operation order with exp / log / expm1 evaluated in
# fp64 and rounded once. The same in numpy: fp32 scalars, np.float64 transcendentals, one rounding.

def _cr(fn, v):
    return f32(fn(np.float64(v)))


class FlowCtlOracle:
    def __init__(self, shift, time_scale):
        self.s, self.m1, self.ts = f32(shift), f32(shift - 1.), f32(time_scale)

    def sigma(self, t):
        return (self.s * t) / (f32(1) + self.m1 * t)

    def marg(self, t):
        t = f32(t)
        sg = self.sigma(t)
        ae = f32(1) - sg
        la = _cr(np.log, ae)
        return dict(t=t, sigma=sg, alpha_e=ae, la=la, lam=la - _cr(np.log, sg), alpha=_cr(np.exp, la))

    def inv(self, lam):
        sg = f32(1) / (f32(1) + _cr(np.exp, lam))
        return sg / (self.s - self.m1 * sg)

    def first(self, pp, ms, mt):
        h = mt["lam"] - ms["lam"]
        if pp:
            return mt["sigma"] / ms["sigma"], -(mt["alpha"] * _cr(np.expm1, -h))
        return _cr(np.exp, mt["la"] - ms["la"]), -(mt["sigma"] * _cr(np.expm1, h))

    def plan2(self, pp, taylor, s, lam_s, hstep):
        """Order 2 (DPM-Solver-12): t, the three evaluation times and input times, coefficient blocks 0..2."""
        t = self.inv(f32(lam_s) + f32(hstep))
        ms, mt = self.marg(s), self.marg(t)
        h = mt["lam"] - ms["lam"]
        r1 = f32(0.5)
        s1 = self.inv(ms["lam"] + r1 * h)
        m1 = self.marg(s1)
        a, c0 = self.first(pp, ms, mt)
        if pp:
            a1, c01 = m1["sigma"] / ms["sigma"], -(m1["alpha"] * _cr(np.expm1, -r1 * h))
            phi_1 = _cr(np.expm1, -h)
            af, bf = mt["sigma"] / ms["sigma"], mt["alpha"] * phi_1
            c1f = (f32(1) / r1) * (mt["alpha"] * (phi_1 / h + f32(1))) if taylor else -((f32(0.5) / r1) * bf)
        else:
            a1, c01 = _cr(np.exp, m1["la"] - ms["la"]), -(m1["sigma"] * _cr(np.expm1, r1 * h))
            phi_1 = _cr(np.expm1, h)
            af, bf = _cr(np.exp, mt["la"] - ms["la"]), mt["sigma"] * phi_1
            c1f = -((f32(1) / r1) * (mt["sigma"] * (phi_1 / h - f32(1)))) if taylor else -((f32(0.5) / r1) * bf)
        z = f32(0)
        blocks = [[a, c0, z, z, z, z, z, z, z, ms["alpha_e"], ms["sigma"]],
                  [a1, c01, z, z, z, z, z, z, z, ms["alpha_e"], ms["sigma"]],
                  [af, -bf, c1f, z, f32(1), z, z, z, z, m1["alpha_e"], m1["sigma"]]]
        tt = [f32(s), s1, f32(s)]
        return t, tt, [self.ts * self.sigma(v) for v in tt], blocks


def _bits(v):
    return np.asarray(v, dtype=f32).view(np.uint32).tolist()


@pytest.mark.parametrize("shift", [1.0, 3.0, 1.15])
@pytest.mark.parametrize("pp,taylor", [(True, False), (True, True), (False, False), (False, True)])
def test_device_controller_words_match_the_once_rounded_oracle(cuda_backend, shift, pp, taylor):
    """State words, coefficient blocks and time labels along a seeded trajectory of accepted and rejected steps, from
    the start of the time range to its end."""
    import dpm_solver_b200 as new
    ns = new.NoiseScheduleFlow(shift=shift, time_scale=1000.0)
    o = FlowCtlOracle(shift, 1000.0)
    t_0, theta, t_err = 1e-3, 0.9, 1e-5
    ctl = cuda_backend.adaptive_controller(ns, torch.device("cuda:0"), order=2, predict_x0=pp, taylor=taylor, t_0=t_0,
                                           theta=theta, t_err=t_err, discrete_input=True)
    ctl.init(ns.T, 0.05)
    s, lam_s, lam_0, h = f32(ns.T), o.marg(ns.T)["lam"], o.marg(t_0)["lam"], f32(0.05)
    rng = np.random.default_rng(int(shift * 100) + 2 * pp + taylor)
    near = 0
    for it in range(400):
        st = ctl.state.cpu().numpy()
        assert _bits(st[:4]) == _bits([s, lam_s, lam_0, h]), (it, st[:4], s, lam_s, lam_0, h)
        if st.view(np.int32)[6]:
            break
        ctl.plan()
        t, tt, tin, blocks = o.plan2(pp, taylor, s, lam_s, h)
        got_t = ctl.state.cpu().numpy()[4]
        times, coef = ctl.times.cpu().numpy(), ctl.coef.cpu().numpy()
        if _bits(got_t) != _bits(t):
            # the fp64 libm of the device and of the host may differ in the last place of a double: at an fp32 rounding
            # boundary either neighbour is right, and everything downstream follows the device's choice
            assert abs(int(_bits(got_t)[0]) - int(_bits(t)[0])) <= 1, (it, got_t, t)
            near += 1
            break
        ok = _bits(times) == _bits(tt + tin) and all(_bits(coef[b][:11]) == _bits(blocks[b]) for b in range(3))
        if not ok:
            ulp = max(abs(int(x) - int(y)) for x, y in zip(_bits(np.concatenate([times, coef[:3, :11].ravel()])),
                                                              _bits(tt + tin + sum(blocks, []))))
            assert ulp <= 1, (it, times, tt, tin, coef[:3, :11], blocks)
            near += 1
        E = f32(rng.choice([0.3, 0.8, 1.0, 1.7, 0.05]))
        ctl.E.fill_(float(E))
        ctl.decide()
        if E <= 1:
            s, lam_s = t, o.marg(t)["lam"]
        grow = f32(np.float64(E) ** (-1.0 / 2))
        h = min((f32(theta) * h) * grow, lam_0 - lam_s)
    else:
        raise AssertionError("the trajectory did not end")
    assert it >= 5 and near <= 2, (it, near)


@needs_ref
@pytest.mark.parametrize("algo", ["dpmsolver++", "dpmsolver"])
@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("guidance", ["none", "scalar"])
def test_adaptive_on_the_device_follows_the_host_controller(cuda_backend, algo, order, guidance):
    x = seeded((3, 4, 16, 16), 25)
    kw = dict(order=order, method="adaptive", atol=0.05, rtol=0.1)
    res = []
    for where in ("device", "host"):
        ps = _product(True, algo, guidance, False)
        ps.adaptive_controller = where
        with mock.patch("builtins.print") as pr:
            y = ps.sample(x.cuda(), **kw)
            res.append((pr.call_args[0][-1], y.cpu().double()))
    assert res[0][0] == res[1][0], (res[0][0], res[1][0])
    # (the bound of the existing device-controller tests: the host libm differs from the once-rounded values in the last ulp)
    assert float((res[0][1] - res[1][1]).abs().max() / res[1][1].abs().max()) <= 1e-4
