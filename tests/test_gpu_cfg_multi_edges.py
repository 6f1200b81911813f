"""The multi-condition step kernels (dpm_step_multi) and dpm_replicate at IEEE edges, on every dispatch path and tuning.

Operands come from tests/step_edges.py: NaN, +-inf, -0, subnormals, numerators at the range guard of the constant
division and divisors on both sides of recip_div_ok, scattered into x, xe, m1, m2, e_uncond and every e_conds[k], with
scales drawn from {1, 0, -0, -1, 3.5, 7.5, NaN, inf}. K = 2, 3, 4, every form, parameterisation and threshold layout
(none, per packet, per element) run on the FAST and generic k_step_multi, tails, views offset by 1, 3, 4 and 8 elements
(on x, on one e_conds[k] only or on one replica only), dev_coef launches, channels_last tensors and the dtype pairs only
k_step_multi_scalar serves. m_out, out and every replica must equal MultiOracle (tests/test_cfg_multi.py; valid at
these edges by tests/test_cfg_multi_edges_vs_reference.py) with NaN in the same places and every other element
bit-identical, and every replica must equal out.

A Python mirror of step_multi_impl names the kernels of every launch; the test tallies (K, kernel, division site,
fallback) and requires the rarely reached ones, and torch.profiler confirms the mirror. The tile loop is run across
thousands of CTAs and several tiles per CTA at every tuning, and dpm_replicate past one pass of its grid."""
import dataclasses
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest
import torch

from dpm_solver_b200._lib import FORM_NONE, FORM_SS3T, PARAM_NOISE, PARAM_SCORE
from dpm_solver_b200.ops import StepArgs
from step_edges import (DIV_OK, DIV_REFUSED, GUARD, GUARD_TINY, PATTERNS, THR_EXTRA, assert_bits_equal, lanes,
                        recip_div_ok, scatter_edges, solve)
from test_cfg_multi import MultiOracle

pytestmark = pytest.mark.gpu
f32 = np.float32
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
CNAME = {F32: "float", BF16: "__nv_bfloat16", F16: "__half"}
PAIRS = [(F32, F32), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32)]   # (model, state) of k_step_multi
SCALAR_PAIRS = [(BF16, F16), (F16, BF16), (F32, BF16), (F32, F16)]       # k_step_multi_scalar only
PATHS = ("direct", "tail", "unaligned", "dev_coef", "cl", "ragged")
OFFSETS = [(k, where) for k in (1, 3, 4, 8) for where in ("x", "ec", "rep")]
ORDINARY = [0.9, -0.3, 0.2, 0.1, 1.5, 0.7, 0.4, 0.6, -1.1]
THRESHOLDS = DIV_OK + DIV_REFUSED + THR_EXTRA + [f32(1.3), f32(0.6), f32(2.5)]
SCALES = [1.0, 0.0, -0.0, -1.0, 3.5, 7.5, float("nan"), float("inf")]
FINITE = [s for s in SCALES if np.isfinite(s)]
COEF_NAMES = ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e")


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def _pick(rng, seq):
    return seq[int(rng.integers(len(seq)))]


def _offset(t, k):
    """t as a view k elements into a fresh storage."""
    buf = torch.empty(t.numel() + k, dtype=t.dtype, device=t.device)
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


# ---- the dispatch, mirrored -------------------------------------------------------------------------------------
def _aligned(t, dt):
    return t.data_ptr() % (32 if dt == F32 else 16) == 0


def mirror_multi(d, md, sd, n):
    """The kernels one launch runs, following capi.cu step_multi_impl (build_params, all_aligned plus every e_conds[k]
    and replica), fast_path_ok, with_packet_pair and the scalar tail. d: the StepArgs handed to the backend."""
    form = d.form
    need_alpha, need_w4 = d.predict_x0, form == FORM_SS3T
    fast_div = (not need_alpha or recip_div_ok(d.alpha_e)) and (not need_w4 or recip_div_ok(d.w4))
    ps = d.per_sample
    pkps = ps // 8 if ps % 8 == 0 else 0
    fast = (not (form == FORM_SS3T and not fast_div) and d.param == PARAM_NOISE and (not d.predict_x0 or fast_div)
            and not (d.thr is not None and pkps == 0))
    use_xe = d.predict_x0 or d.param in (1, 2)
    state = ([d.x] if form != FORM_NONE else []) + ([d.xe if d.xe is not None else d.x] if use_xe else [])
    state += [t for t, f in ((d.m1, (2, 3, 4, 5, 6)), (d.m2, (3, 5, 6))) if form in f]
    state += list(d.replicas or ()) if form != FORM_NONE else []
    ok = all(_aligned(t, sd) for t in state) and all(_aligned(t, md) for t in (d.e_uncond,) + tuple(d.e_conds))
    scalar = ("scalar",)
    if n // 8 > 0 and ok and d.coef_dev is None and (md, sd) in PAIRS:
        return [("multi", CNAME[md], CNAME[sd], form, fast)] + ([scalar] if n % 8 else []), fast_div
    return [scalar], fast_div


def kernel_label(k, dev_coef):
    if dev_coef:
        return "scalar(dev_coef)"
    return ("multi-fast" if k[4] else "multi-generic") if k[0] == "multi" else "scalar"


def kernel_name(k):
    if k[0] == "multi":
        return "k_step_multi<%s,%s,%d,%s>" % (k[1], k[2], k[3], "true" if k[4] else "false")
    return "k_step_multi_scalar"


# ---- one launch ---------------------------------------------------------------------------------------------------
def build_case(spec):
    """StepArgs on the host for one seeded case, plus what the checks need to know about it."""
    rng = np.random.default_rng(spec["seed"])
    K, path, form, div, md, sd = spec["K"], spec["path"], spec["form"], spec["div"], spec["md"], spec["sd"]
    B, ps = {"tail": (3, 67), "ragged": (6, 12)}.get(path, (4, 64))
    n = B * ps
    param = PARAM_NOISE if rng.random() < 0.5 else int(rng.integers(1, 4))
    px0 = rng.random() < 0.7 or path == "ragged"
    ss3t_plant = form == FORM_SS3T and md == sd == F32 and div == "ok" and path != "ragged" and rng.random() < 0.7
    if ss3t_plant:                    # the numerators of the w4 divisions are planted below on the FAST kernel's path
        param, px0 = PARAM_NOISE, False
    coef = {k: f32(_pick(rng, ORDINARY)) for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3")}
    alpha, w4 = f32(_pick(rng, DIV_OK + [f32(0.8)])), f32(_pick(rng, DIV_OK + [f32(0.3)]))
    if div == "refused":
        which = _pick(rng, [w for w in ("alpha", "w4") if (w == "alpha" and px0) or (w == "w4" and form == FORM_SS3T)]
                      or ["none"])
        if which == "alpha":
            alpha = _pick(rng, DIV_REFUSED)
        elif which == "w4":
            w4 = _pick(rng, DIV_REFUSED)
    scales = tuple(float(_pick(rng, SCALES if rng.random() < 0.2 and not ss3t_plant else FINITE)) for _ in range(K))
    finite = all(np.isfinite(scales))
    a = StepArgs(form=form, n_model=2, param=param, predict_x0=px0, c0_on_old=bool(rng.random() < 0.5),
                 alpha_e=float(alpha), sigma_e=float(_pick(rng, [0.6, 0.03, 1.0])), w4=float(w4), want_m_out=True,
                 state_dtype=sd, per_sample=ps, scales=scales, **{k: float(v) for k, v in coef.items()})
    streams, dtypes = {}, {}

    def add(name, dt, scale=1.0):
        streams[name] = (rng.standard_normal(n) * scale).astype(f32)
        dtypes[name] = dt
    if form != FORM_NONE:
        add("x", sd)
    add("e_uncond", md)
    ecs = ["ec%d" % k for k in range(K)]
    for k, e in enumerate(ecs):
        add(e, md, 1.0 + 0.2 * k)
    if px0 or param in (1, 2):
        if form == FORM_NONE or rng.random() < 0.4:
            add("xe", sd)
    if form in (2, 3, 4, 5, 6):
        add("m1", sd)
    if form in (3, 5, 6):
        add("m2", sd)
    scatter_edges(streams, dtypes, rng)
    xe_name = "xe" if "xe" in streams else "x"
    fp32 = sd == F32 and md == F32 and finite
    npk = n // 8

    def plant_packets(k):
        return [(pk, lanes(_pick(rng, PATTERNS), rng)) for pk in rng.choice(npk, size=min(k, npk), replace=False)]

    def zero_outputs(i, v=0.0):
        for s in ["e_uncond"] + ecs:
            streams[s][i] = v
    # x0's numerator xe - sigma*eps at the guard: every network output 0 in those lanes (eps = 0 for finite scales)
    if fp32 and px0 and param in (PARAM_NOISE, PARAM_SCORE):
        for pk, ls in plant_packets(3):
            for l in ls:
                i = pk * 8 + l
                zero_outputs(i)
                streams[xe_name][i] = GUARD[i % len(GUARD)]
    # per-sample thresholds; the clamp division's numerators at the guard in a sample with an accepted threshold
    thr = None
    if px0 and (path == "ragged" or rng.random() < 0.6):
        thr = np.array([_pick(rng, THRESHOLDS) for _ in range(B)], dtype=f32)
        if fp32 and param in (PARAM_NOISE, PARAM_SCORE):
            b = int(rng.integers(B))
            thr[b] = _pick(rng, DIV_OK + [f32(1.3)])
            for pk, ls in plant_packets(3 * B):
                if pk * 8 // ps != b:
                    continue
                for l in ls:
                    i = pk * 8 + l
                    t = GUARD_TINY[i % len(GUARD_TINY)]
                    xe = solve(lambda v: v / alpha, t, f32(t * alpha))
                    if xe is None:
                        continue
                    zero_outputs(i)
                    streams[xe_name][i] = xe
    # SS3T: n1 = -(w3*(w1*T0)) and n2 = 2*(w1*T0) at the guard with m1 = m2 = 0; T0 = eps when every output is T0
    if fp32 and form == FORM_SS3T and param == PARAM_NOISE and not px0:
        w1, w3 = coef["w1"], coef["w3"]
        cnt = spec["seed"]
        for pk, ls in plant_packets(8):
            for l in ls:
                i = pk * 8 + l
                cnt += 1
                t = GUARD[cnt % len(GUARD)]
                if rng.random() < 0.5:
                    T = solve(lambda v: f32(2) * (w1 * v), t, f32(t / 2 / w1))
                else:
                    D = solve(lambda v: -(w3 * v), t, f32(-t / w3))
                    T = None if D is None else solve(lambda v: w1 * v, D, f32(D / w1))
                if T is None:
                    continue
                streams["m1"][i] = streams["m2"][i] = 0.0
                zero_outputs(i, T)
    shape = (B, 4, 4, 4) if path == "cl" else (B, ps)
    host = {k: torch.from_numpy(v).to(dtypes[k]).reshape(shape) for k, v in streams.items()}
    for k in ("x", "xe", "m1", "m2", "e_uncond"):
        if k in host:
            setattr(a, k, host[k])
    a.e_conds = tuple(host[e] for e in ecs)
    a.e_cond = a.e_conds[0]
    if xe_name == "x" and (px0 or param in (1, 2)):
        a.xe = a.x
    if thr is not None:
        a.thr = torch.from_numpy(thr)
    if path == "dev_coef":
        a.coef_dev = torch.tensor([getattr(a, k) for k in COEF_NAMES] + [0.0] * 5, dtype=torch.float32)
    return a, dict(n=n, B=B, ps=ps)


def to_device(a, spec):
    """The StepArgs the backend gets: tensors on the GPU, offset or channels_last as the path asks, NaN-filled
    replicas, and with dev_coef host scalars the launch must not read."""
    d = dataclasses.replace(a)
    cl = spec["path"] == "cl"
    k, where = spec.get("offset", (0, None))
    rng = np.random.default_rng(spec["seed"] + 1)

    def dev(t, shift=0):
        t = t.cuda()
        if cl:
            t = t.contiguous(memory_format=torch.channels_last)
        return _offset(t, shift) if shift else t
    for f in ("x", "xe", "m1", "m2", "e_uncond"):
        t = getattr(a, f)
        if t is not None:
            setattr(d, f, dev(t, k if (where == "x" and f == "x") else 0))
    if a.xe is not None and a.xe is a.x:
        d.xe = d.x
    j = int(rng.integers(len(a.e_conds)))
    d.e_conds = tuple(dev(e, k if (where == "ec" and i == j) else 0) for i, e in enumerate(a.e_conds))
    d.e_cond = d.e_conds[0]
    if a.thr is not None:
        d.thr = a.thr.cuda()
    if a.form != FORM_NONE:
        ref = d.x
        reps = []
        for i in range(len(a.e_conds)):
            r = torch.full_like(ref, float("nan"))
            reps.append(_offset(r, k) if (where == "rep" and i == j) else r)
        d.replicas = tuple(reps)
    if a.coef_dev is not None:
        d.coef_dev = a.coef_dev.cuda()
        for name in COEF_NAMES:
            setattr(d, name, -3.0 * getattr(a, name) + 0.25)      # the launch must read the device block
    return d


def run_case(be, spec, tally=None, hits=None):
    a, info = build_case(spec)
    d = to_device(a, spec)
    gm, go = be.step(d)
    with np.errstate(all="ignore"):
        wm, wo = MultiOracle().step(a)
    what = "%s %s" % (spec, dict(param=a.param, px0=a.predict_x0, alpha=a.alpha_e, w4=a.w4, scales=a.scales,
                                 thr=None if a.thr is None else a.thr.tolist()))
    assert_bits_equal(gm, wm, "m_out of " + what)
    assert (go is None) == (wo is None), what
    if go is not None:
        assert_bits_equal(go, wo, "out of " + what)
        iv = torch.int32 if go.element_size() == 4 else torch.int16
        for r in d.replicas:
            assert torch.equal(r.view(iv), go.view(iv)), "replica of " + what
    kernels, fast_div = mirror_multi(d, spec["md"], spec["sd"], info["n"])
    if tally is not None:
        _tally(tally, hits, spec, a, kernels, fast_div, gm)
    return kernels


# ---- tallies ------------------------------------------------------------------------------------------------------
def _tally(tally, hits, spec, a, kernels, fast_div, gm):
    K = len(a.e_conds)
    dev_coef = a.coef_dev is not None
    lab = kernel_label(kernels[0], dev_coef)
    fast = lab == "multi-fast"
    tally[(K, lab, "launch", "")] += 1
    if len(kernels) > 1:
        tally[(K, "scalar", "tail", "")] += 1
    if a.predict_x0:
        tally[(K, lab, "alpha", "recip" if fast else ("refused" if not recip_div_ok(a.alpha_e) else "ieee"))] += 1
    if a.form == FORM_SS3T:
        tally[(K, lab, "w4", "recip" if fast_div and not dev_coef else "ieee")] += 1
    if a.thr is not None:
        for s in a.thr.numpy():
            kind = "recip" if recip_div_ok(s) else ("ieee-finite" if np.isfinite(s) else "ieee-nonfinite")
            tally[(K, lab, "thr", kind if fast else "ieee")] += 1
    # numerators of each division site and the fp64 check of the quotients (fp32 streams, finite scales)
    if a.state_dtype != F32 or a.e_cond.dtype != F32 or not all(np.isfinite(a.scales)):
        return
    with np.errstate(all="ignore"):
        if a.param not in (PARAM_NOISE, PARAM_SCORE):
            return
        conv = (lambda v: (-f32(a.sigma_e)) * v) if a.param == PARAM_SCORE else (lambda v: v)
        eu = conv(a.e_uncond.numpy().reshape(-1))
        eps = eu
        for s, e in zip(a.scales, a.e_conds):
            eps = eps + f32(s) * (conv(e.numpy().reshape(-1)) - eu)
        if a.predict_x0:
            xe = (a.xe if a.xe is not None else a.x).numpy().reshape(-1)
            num = xe - f32(a.sigma_e) * eps
            x0 = (num.astype(np.float64) / np.float64(f32(a.alpha_e))).astype(f32)
            want = x0
            if a.thr is not None:
                s = np.repeat(a.thr.numpy(), a.per_sample)
                c = np.where(x0 > s, s, np.where(x0 < -s, -s, x0))
                want = (c.astype(np.float64) / s.astype(np.float64)).astype(f32)
                acc = np.array([recip_div_ok(v) for v in s])
                if fast:
                    for t in GUARD_TINY:
                        hits[("thr", float(t))] += int(((c == t) & acc).sum())
            if fast:
                for t in GUARD:
                    hits[("alpha", float(t))] += int((num == t).sum())
            if a.form == FORM_NONE:
                got = gm.cpu().numpy().reshape(-1)
                fin = np.isfinite(got)
                assert (got[fin].view(np.uint32) == want[fin].view(np.uint32)).all(), \
                    ("fp64 quotient", spec, int((got[fin] != want[fin]).sum()))
                tally[("fp64 checked", "thr" if a.thr is not None else "alpha")] += int(fin.sum())
        elif a.form == FORM_SS3T and fast and a.param == PARAM_NOISE:
            m1, m2 = a.m1.numpy().reshape(-1), a.m2.numpy().reshape(-1)
            D10, D11 = f32(a.w0) * (m1 - m2), f32(a.w1) * (eps - m2)
            n1, n2 = f32(a.w2) * D10 - f32(a.w3) * D11, f32(2) * (D11 - D10)
            for t in GUARD:
                hits[("w4", float(t))] += int((n1 == t).sum() + (n2 == t).sum())


# ---- the case list ------------------------------------------------------------------------------------------------
def case_specs():
    specs, seed = [], 0
    for K in (2, 3, 4):
        for path in PATHS:
            for form in range(7):
                for div in ("ok", "refused"):
                    if path == "unaligned":
                        variants = [dict(md=PAIRS[i % 5][0], sd=PAIRS[i % 5][1], offset=o) for i, o in enumerate(OFFSETS)]
                    else:
                        pairs = PAIRS + (SCALAR_PAIRS if path == "direct" else [])
                        variants = [dict(md=md, sd=sd) for md, sd in pairs]
                    for v in variants:
                        seed += 1
                        specs.append(dict(K=K, path=path, form=form, div=div, seed=70000 + seed, **v))
    return specs


REQUIRED = [(K, lab, site, fb) for K in (2, 3, 4) for lab, site, fb in (
    ("multi-fast", "alpha", "recip"), ("multi-fast", "thr", "recip"), ("multi-fast", "thr", "ieee-finite"),
    ("multi-fast", "thr", "ieee-nonfinite"), ("multi-fast", "w4", "recip"),
    ("multi-generic", "alpha", "refused"), ("multi-generic", "w4", "ieee"),
    ("scalar", "thr", "ieee"), ("scalar(dev_coef)", "launch", ""), ("scalar", "tail", ""))]
REQUIRED += [("fp64 checked", "alpha"), ("fp64 checked", "thr")]
REQUIRED_HITS = ([("alpha", float(t)) for t in GUARD] + [("thr", float(t)) for t in GUARD_TINY]
                 + [("w4", float(t)) for t in GUARD])


def test_multi_step_kernels_at_ieee_edges(cuda_backend):
    tally, hits = Counter(), Counter()
    specs = case_specs()
    for spec in specs:
        run_case(cuda_backend, spec, tally, hits)
    print("\n%d edge-valued multi-condition launches; path tally:" % len(specs))
    for k, v in sorted(tally.items(), key=str):
        print("  %-60s %d" % (k, v))
    print("numerator hits:", dict(sorted(hits.items(), key=str)))
    missing = [k for k in REQUIRED if tally[k] == 0] + [k for k in REQUIRED_HITS if hits[k] == 0]
    assert not missing, missing


def profile_mirror():
    """The dispatch mirror against torch.profiler's kernel names: one launch for every kernel instantiation the cases
    reach and for every (kernel kind, tail) combination, one profiler session each."""
    from dpm_solver_b200 import ops
    from torch.profiler import ProfilerActivity, profile
    be = ops.CudaBackend()
    chosen, seen = [], set()
    for spec in case_specs():
        a, info = build_case(spec)
        ks, _ = mirror_multi(to_device(a, spec), spec["md"], spec["sd"], info["n"])
        dc = a.coef_dev is not None
        new = {(kernel_name(k), dc) for k in ks} | {(kernel_label(ks[0], dc), len(ks))}
        if not new <= seen:
            chosen.append(spec)
            seen |= new
    kinds = {k for k in seen if isinstance(k[1], int)}
    assert {("multi-fast", 1), ("multi-fast", 2), ("multi-generic", 1), ("multi-generic", 2), ("scalar", 1),
            ("scalar(dev_coef)", 1)} <= kinds and len(chosen) >= 70, (kinds, len(chosen))
    # one profiler session for every launch (sessions opened one after another were seen to record no kernels): the
    # step kernels run in launch order on one stream, so the recorded sequence must be the mirror's, launch by launch
    want, owner = [], []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for spec in chosen:
            ks = run_case(be, spec)
            want += [kernel_name(k) + ("(" if k[0] == "scalar" else "") for k in ks]
            owner += [spec] * len(ks)
        torch.cuda.synchronize()
    ran = [e.name.replace(" ", "") for e in sorted((e for e in prof.events() if "k_step_multi" in e.name),
                                                   key=lambda e: e.time_range.start)]
    assert len(ran) == len(want), (len(ran), len(want))
    for spec, w, r in zip(owner, want, ran):
        assert w in r, (spec, w, r)
    print("%d profiled launches match the mirror" % len(chosen))


def test_mirror_names_the_kernel_that_ran():
    """profile_mirror() in a child process of its own, in one profiler session: sessions opened after many others in
    one process were seen to record no kernels (tests/test_gpu_step_edges.py profiles in this process too, and a child
    that opened one session per launch once recorded nothing in one of them), so neither test may leave its profiler
    state to the other."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path[:0] = %r; import test_gpu_cfg_multi_edges as t; t.profile_mirror()"
            % [root, os.path.join(root, "tests"), os.path.join(root, "tests", "golden")])
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-4000:], r.stderr[-4000:])
    print(r.stdout.strip().splitlines()[-1])


# ---- the tile loop across CTAs, at every tuning -------------------------------------------------------------------
def _tuning_case(name):
    """Large launches: 2^25 elements plus a ragged tail. With 256 threads and 32 CTAs per SM some CTA runs at least
    two tiles; fewer threads or CTAs per SM only add tiles per CTA."""
    g = torch.Generator(device="cuda").manual_seed(5)
    if name == "fast-inplace":        # FAST, MS3, x updated in place (a CTA that re-ran a tile would read its output)
        K, md, sd, form, ps, thr = 3, BF16, BF16, 5, 4100, False
    elif name == "fast-thr":          # FAST, per-packet thresholds
        K, md, sd, form, ps, thr = 2, F32, F32, 4, 4096, True
    else:                             # ragged samples: generic body with per-element thresholds, scalar tail
        K, md, sd, form, ps, thr = 4, F16, F32, 6, 1000 * 8 + 3, True
    B = (1 << 25) // ps + 1
    n = B * ps
    mk = lambda dt, scale=1.0: (torch.randn(n, device="cuda", generator=g) * scale).to(dt)
    x = mk(sd)
    a = StepArgs(form=form, n_model=2, x=x, xe=x, e_uncond=mk(md), predict_x0=True, alpha_e=0.83, sigma_e=0.55,
                 state_dtype=sd, want_m_out=True, per_sample=ps, scales=tuple(SCALES[3:3 + K]) if K < 4 else
                 (7.5, -1.0, 0.0, 3.5), a=0.94983894, c0=0.0897649, c1=-0.04488245, c2=0.0021, w0=0.9766731,
                 w1=1.0613433, w2=0.4912, w3=0.4796, w4=0.3)
    a.e_conds = tuple(mk(md, 1.0 + 0.2 * k) for k in range(K))
    a.e_cond = a.e_conds[0]
    if form in (2, 3, 4, 5, 6):
        a.m1 = mk(sd)
    if form in (3, 5, 6):
        a.m2 = mk(sd)
    if thr:
        a.thr = torch.rand(B, device="cuda", generator=g) * 0.3 + 0.3     # distinct per sample, clamps most x0
    return a, name == "fast-inplace"


def _run_tuned(be, a, inplace, variant, threads, ctas):
    d = dataclasses.replace(a)
    if inplace:
        d.x = d.xe = a.x.clone()
        d.out = d.x
    d.replicas = tuple(torch.empty_like(a.x) for _ in a.e_conds)
    be.set_tuning(variant, threads, ctas)
    try:
        m, o = be.step(d)
    finally:
        be.set_tuning(2, 0, 0)
    return m, o, d.replicas


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


@pytest.mark.parametrize("name", ["fast-inplace", "fast-thr", "ragged-thr"])
def test_multi_step_tuning_invariance_across_ctas(cuda_backend, name):
    a, inplace = _tuning_case(name)
    m0, o0, r0 = _run_tuned(cuda_backend, a, inplace, 2, 0, 0)
    for r in r0:
        assert torch.equal(_bits(r), _bits(o0))
    host = dataclasses.replace(a, x=a.x.cpu(), xe=a.x.cpu(), e_uncond=a.e_uncond.cpu(), e_cond=a.e_cond.cpu(),
                               e_conds=tuple(e.cpu() for e in a.e_conds), m1=None if a.m1 is None else a.m1.cpu(),
                               m2=None if a.m2 is None else a.m2.cpu(), thr=None if a.thr is None else a.thr.cpu())
    with np.errstate(all="ignore"):
        wm, wo = MultiOracle().step(host)
    assert_bits_equal(m0, wm, "m_out of the default tuning")
    assert_bits_equal(o0, wo, "out of the default tuning")
    del wm, wo, host
    for variant, threads, ctas in [(2, t, c) for t in (0, 32, 64, 128, 256, 512) for c in (0, 1, 2, 4, 32)] + \
                                  [(1, 0, 0)]:
        m, o, reps = _run_tuned(cuda_backend, a, inplace, variant, threads, ctas)
        assert torch.equal(_bits(m), _bits(m0)), (variant, threads, ctas)
        assert torch.equal(_bits(o), _bits(o0)), (variant, threads, ctas)
        for r in reps:
            assert torch.equal(_bits(r), _bits(o0)), (variant, threads, ctas)
        del m, o, reps


# ---- dpm_replicate past one pass of its grid ------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F32, BF16, F16])
def test_replicate_beyond_one_grid_pass(cuda_backend, dt):
    """k_replicate's grid is sm_count*16 CTAs of 256 threads, one 16-byte word each per pass: sizes of 2.5 passes run
    the stride loop three times. The vector kernel, the copy fallback (an unaligned view, a size that is not a whole
    number of words) and channels_last, each equal to torch.cat byte for byte."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_word = 16 // torch.empty(0, dtype=dt).element_size()
    n = sms * 16 * 256 * per_word * 5 // 2                   # whole words, 2.5 passes
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n + 1, device="cuda", generator=g).to(dt)
    cases = {"vector": x[:n].view(-1, 256), "unaligned": x[1:].view(-1, 256),
             "bytes%16": x[:n - 1].view(-1, 1), "channels_last": x[:n].view(-1, 8, 8, 4).contiguous(
                 memory_format=torch.channels_last)}
    assert cases["vector"].data_ptr() % 16 == 0 and n // per_word > sms * 16 * 256 * 2
    for route, v in cases.items():
        for copies in (1, 2, 5):
            got = cuda_backend.replicate(v, copies)
            want = torch.cat([v] * copies)
            assert got.shape == want.shape and got.stride() == want.stride(), (route, copies)
            assert torch.equal(_bits(got), _bits(want)), (route, copies)
            del got, want
