"""The fused step kernels at IEEE edges, on every dispatch path, against the numpy executor.

Operands come from tests/step_edges.py: NaN, +-inf, -0, subnormals, overflowing updates, fp16 results at the
round-to-infinity boundary, numerators at the range guard of the constant division and divisors on both sides of
recip_div_ok, placed per packet in lane 0, lane 7, all lanes or mixed. Every step family (plain, reference rounding,
guidance rescale, per-sample guidance), form, dtype pair, parameterisation and threshold layout runs on the direct
FAST and generic kernels, the TMA ring, tails, unaligned views, ragged samples and dev_coef launches. m_out, out and
out2 must equal the executor's with NaN in the same places and every other element bit-identical.

A Python mirror of the dispatch (fast_path_ok, recip_div_ok, pick_direct, the TMA conditions) names the kernel of
every launch; the test tallies (family, kernel, division site, fallback) and requires the rarely reached ones,
among them the SS3T kernels without network outputs on IEEE division and the finite refused threshold of the FAST
kernels. torch.profiler confirms the mirror on a sample of launches. Division results are also checked against
fp64: fl32(float64(num) / float64(d)) is the correctly rounded fp32 quotient (53 >= 2*24 + 2)."""
import dataclasses
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest
import torch

from dpm_solver_b200._lib import (FORM_LIN1, FORM_NONE, FORM_SS3T, PARAM_NOISE, PARAM_SCORE)
from dpm_solver_b200.ops import StepArgs
from step_edges import (DIV_OK, DIV_REFUSED, F16_INF_EDGE, F16_MAX, GUARD, GUARD_TINY, THR_EXTRA, assert_bits_equal,
                        lanes, PATTERNS, recip_div_ok, scatter_edges, solve)
from test_cfg_per_sample import GuidedOracle

pytestmark = pytest.mark.gpu
f32 = np.float32
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
CODE = {F32: 0, BF16: 1, F16: 2}
CNAME = {F32: "float", BF16: "__nv_bfloat16", F16: "__half"}
PAIRS = [(F32, F32), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32)]     # (model, state) of the packet kernels
MIXED = (BF16, F16)                                                          # served by the scalar kernel only
FAMILIES = ("plain", "rnd", "rs", "pg")
PATHS = ("direct", "tma", "tail", "unaligned", "ragged", "dev_coef")
ORDINARY = [0.9, -0.3, 0.2, 0.1, 1.5, 0.7, 0.4, 0.6, -1.1]
THRESHOLDS = DIV_OK + DIV_REFUSED + THR_EXTRA + [f32(1.3), f32(0.6), f32(2.5)]
RATIOS = [0.0, float("nan"), float("inf"), 1.0, 0.8, 1.7]
SCALES = [1.0, 0.0, -1.0, float("nan"), float("inf"), 3.5, 7.5]


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


# ---- the dispatch, mirrored -------------------------------------------------------------------------------------
def mirror(a, md, sd, n, aligned, variant):
    """The kernels one launch runs, as (kind, template arguments) tuples, following capi.cu step_impl, fast_path_ok,
    pick_direct and launch_step_tma."""
    ne, form = a.n_model, a.form
    need_alpha, need_w4 = ne >= 1 and a.predict_x0, form == FORM_SS3T
    fast_div = (not need_alpha or recip_div_ok(a.alpha_e)) and (not need_w4 or recip_div_ok(a.w4))
    ps = a.per_sample
    pkps = ps // 8 if ps % 8 == 0 else 0
    per_sample_data = a.thr is not None or a.ratio is not None or a.guidance_b is not None
    if form == FORM_SS3T and not fast_div:
        fast = False
    elif ne == 0:
        fast = True
    else:
        fast = a.param == PARAM_NOISE and (not a.predict_x0 or fast_div) and not (per_sample_data and pkps == 0)
    rnd, rs, pg = a.raw_round != 0, a.ratio is not None, a.guidance_b is not None
    te = sd if ne == 0 else md
    scalar = ("scalar", rnd, rs and not pg, pg)
    npk = n // 8
    body = None
    if npk > 0 and aligned and a.coef_dev is None:
        pair_ok = (te, sd) in PAIRS and (ne > 0 or te == sd)
        if variant == 1 and not rnd and not rs and not pg and fast and a.thr is None and pair_ok:
            body = ("tma", CNAME[te], CNAME[sd], ne, form)
        elif pair_ok and not (pg and pkps == 0):
            if pg or rs:
                body = ("direct", CNAME[te], CNAME[sd], 2, form, fast, False, rs and not pg, pg) if ne == 2 else None
            elif rnd:
                ok = sd == F32 and (ne == 0) == (te == F32)
                body = ("direct", CNAME[te], CNAME[sd], ne, form, False, True, False, False) if ok else None
            else:
                body = ("direct", CNAME[te], CNAME[sd], ne, form, fast or (ne == 0 and form != FORM_SS3T),
                        False, False, False)
    if body is None:
        return [scalar], fast_div
    return [body] + ([scalar] if n % 8 else []), fast_div


def kernel_label(k):
    if k[0] == "direct":
        return "direct-fast" if k[5] else "direct-generic"
    return k[0]


def kernel_name(k):
    """The leading template arguments of the kernel's demangled name."""
    b = lambda v: "true" if v else "false"
    if k[0] == "direct":
        return "k_step_direct<%s,%s,%d,%d,%s,%s,%s,%s>" % (k[1], k[2], k[3], k[4], b(k[5]), b(k[6]), b(k[7]), b(k[8]))
    if k[0] == "tma":
        return "k_step_tma<%s,%s,%d,%d>" % k[1:]
    return "k_step_scalar<%s,%s,%s>" % (b(k[1]), b(k[2]), b(k[3]))


# ---- one launch ---------------------------------------------------------------------------------------------------
def _pick(rng, seq):
    return seq[int(rng.integers(len(seq)))]


def _offset(t, k):
    buf = torch.empty(t.numel() + k, dtype=t.dtype, device="cuda")
    v = buf[k:].view(t.shape)
    v.copy_(t)
    return v


def build_case(spec):
    """StepArgs on the host for one seeded case, plus what the checks need to know about it."""
    rng = np.random.default_rng(spec["seed"])
    fam, path, form, ne, div = spec["fam"], spec["path"], spec["form"], spec["ne"], spec["div"]
    md, sd = spec["md"], spec["sd"]
    B, ps = {"tail": (3, 67), "ragged": (6, 12)}.get(path, (4, 64))
    n = B * ps
    param = PARAM_NOISE if (fam == "rnd" or rng.random() < 0.5) else int(rng.integers(1, 4))
    px0 = ne > 0 and (rng.random() < 0.7 or path == "ragged")
    coef = {k: f32(_pick(rng, ORDINARY)) for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3")}
    alpha, w4 = f32(_pick(rng, DIV_OK + [f32(0.8)])), f32(_pick(rng, DIV_OK + [f32(0.3)]))
    if div == "refused":
        which = _pick(rng, [w for w in ("alpha", "w4") if (w == "alpha" and px0) or (w == "w4" and form == FORM_SS3T)]
                      or ["none"])
        if which == "alpha":
            alpha = _pick(rng, DIV_REFUSED)
        elif which == "w4":
            w4 = _pick(rng, DIV_REFUSED)
    a = StepArgs(form=form, n_model=ne, param=param, predict_x0=px0, c0_on_old=bool(rng.random() < 0.5),
                 guidance=float(_pick(rng, [1.0, 3.5, 7.5] if fam != "rnd" else [3.5, 7.5])), alpha_e=float(alpha),
                 sigma_e=float(_pick(rng, [0.6, 0.03, 1.0])), w4=float(w4), want_m_out=ne > 0, state_dtype=sd,
                 per_sample=ps, **{k: float(v) for k, v in coef.items()})
    # streams as fp32 arrays first (edges and planted lanes), cast to their storage type at the end
    streams, dtypes = {}, {}

    def add(name, dt, scale=1.0):
        streams[name] = (rng.standard_normal(n) * scale).astype(f32)
        dtypes[name] = dt
    if form != FORM_NONE:
        add("x", sd)
    if ne == 0:
        add("m0", sd)
    else:
        add("e_cond", md, 1.3)
        if ne == 2:
            add("e_uncond", md)
        if px0 or param in (1, 2):
            if form == FORM_NONE or rng.random() < 0.4:
                add("xe", sd)
    if form in (2, 3, 4, 5, 6):
        add("m1", sd)
    if form in (3, 5, 6):
        add("m2", sd)
    scatter_edges(streams, dtypes, rng)
    xe_name = "xe" if "xe" in streams else "x"
    fp32_plain = fam == "plain" and sd == F32 and (ne == 0 or md == F32)
    planted = Counter()
    npk = n // 8

    def plant_packets(k):
        return [(pk, lanes(_pick(rng, PATTERNS), rng)) for pk in rng.choice(npk, size=min(k, npk), replace=False)]
    # numerators of x0 = (xe - sigma*eps) / alpha at the guard: eps = 0 in those lanes (noise / score networks)
    if fp32_plain and ne > 0 and px0 and param in (PARAM_NOISE, PARAM_SCORE):
        for pk, ls in plant_packets(3):
            for l in ls:
                i = pk * 8 + l
                for s in ("e_cond", "e_uncond"):
                    if s in streams:
                        streams[s][i] = 0.0
                streams[xe_name][i] = GUARD[i % len(GUARD)]
    # per-sample thresholds; the clamp division's numerators at the guard (x0 = +-1e-25 and its neighbours), planted
    # in a sample whose threshold the FAST kernels divide by with the reciprocal
    thr = None
    if ne > 0 and px0 and (path == "ragged" or rng.random() < 0.6):
        thr = np.array([_pick(rng, THRESHOLDS) for _ in range(B)], dtype=f32)
        if fp32_plain and param in (PARAM_NOISE, PARAM_SCORE):
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
                    for s in ("e_cond", "e_uncond"):
                        if s in streams:
                            streams[s][i] = 0.0
                    streams[xe_name][i] = xe
    # SS3T: n1 = -(w3*(w1*T0)) and n2 = 2*(w1*T0) at the guard with m1 = m2 = 0 (so D10 = 0), T0 solved on the host
    if fp32_plain and form == FORM_SS3T and (ne == 0 or (param == PARAM_NOISE and not px0)):
        w1, w3 = coef["w1"], coef["w3"]
        for pk, ls in plant_packets(3):
            for l in ls:
                i = pk * 8 + l
                t = GUARD[i % len(GUARD)]
                if rng.random() < 0.5:
                    T = solve(lambda v: f32(2) * (w1 * v), t, f32(t / 2 / w1))
                else:
                    D = solve(lambda v: -(w3 * v), t, f32(-t / w3))
                    T = None if D is None else solve(lambda v: w1 * v, D, f32(D / w1))
                if T is None:
                    continue
                streams["m1"][i] = streams["m2"][i] = 0.0
                for s in ("m0", "e_cond", "e_uncond"):
                    if s in streams:
                        streams[s][i] = T
    # fp16 state: results on both sides of 65520, the fp16 round-to-infinity boundary
    if sd == F16 and fam == "plain" and form == FORM_LIN1 and ne == 0 and coef["c0"] != 0:
        A, c0 = coef["a"], coef["c0"]
        grid = torch.arange(0, 0x7c00, dtype=torch.int16).view(F16).float().numpy()
        grid = np.concatenate([grid, -grid])
        for pk, ls in plant_packets(2):
            for l in ls:
                i = pk * 8 + l
                side = rng.random() < 0.5
                for free in ("m0", "x"):     # one operand at +-65504, the other searched over every finite fp16
                    fixed = f32(np.sign(A if free == "m0" else c0) * F16_MAX)
                    with np.errstate(all="ignore"):
                        r = A * fixed + c0 * grid if free == "m0" else A * grid + c0 * fixed
                    cand = np.where((r >= F16_INF_EDGE) if side else (r < F16_INF_EDGE), r, np.nan)
                    if np.isnan(cand).all():
                        continue
                    j = np.nanargmin(cand) if side else np.nanargmax(cand)
                    streams[free][i], streams["x" if free == "m0" else "m0"][i] = grid[j], fixed
                    planted["f16 >= 65520" if side else "f16 < 65520"] += 1
                    break
    # RND with 16-bit outputs: a CFG combine whose 16-bit difference overflows
    if fam == "rnd" and ne == 2:
        big = 65504.0 if md == F16 else 3.0e38
        for pk, ls in plant_packets(1):
            streams["e_cond"][pk * 8 + ls], streams["e_uncond"][pk * 8 + ls] = big, -big
    host = {k: torch.from_numpy(v).to(dtypes[k]).reshape(B, ps) for k, v in streams.items()}
    for k, v in host.items():
        setattr(a, k, v)
    if xe_name == "x" and (px0 or param in (1, 2)) and ne > 0:
        a.xe = a.x
    if thr is not None:
        a.thr = torch.from_numpy(thr)
    if fam == "rnd":
        a.raw_round = (CODE[md] if md != F32 else int(rng.integers(1, 3))) | (4 if rng.random() < 0.6 else 0)
    if fam in ("rs", "pg") and (fam == "rs" or rng.random() < 0.5):
        a.ratio = torch.tensor([_pick(rng, RATIOS) for _ in range(B)], dtype=torch.float32)
        a.phi = float(_pick(rng, [0.7, 0.0]))
    if fam == "pg":
        a.guidance_b = torch.tensor([_pick(rng, SCALES) for _ in range(B)], dtype=torch.float32)
    if path == "dev_coef":
        names = ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e")
        a.coef_dev = torch.tensor([getattr(a, k) for k in names] + [0.0] * 5, dtype=torch.float32)
    out2 = form != FORM_NONE and rng.random() < 0.3
    return a, dict(n=n, B=B, ps=ps, out2=out2, planted=planted)


def _to_device(a, path):
    d = dataclasses.replace(a)
    k = 1 if path == "unaligned" else 0
    for f in ("x", "xe", "m0", "m1", "m2", "e_cond", "e_uncond"):
        t = getattr(a, f)
        if t is not None:
            setattr(d, f, _offset(t.cuda(), k) if k else t.cuda())
    if a.xe is not None and a.xe is a.x:
        d.xe = d.x
    for f in ("thr", "ratio", "guidance_b"):
        if getattr(a, f) is not None:
            setattr(d, f, getattr(a, f).cuda())
    if a.coef_dev is not None:
        d.coef_dev = a.coef_dev.cuda()
        for name in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e"):
            setattr(d, name, -3.0 * getattr(a, name) + 0.25)          # the launch must read the device block
    return d


def run_case(be, spec, tally=None, hits=None):
    a, info = build_case(spec)
    n, path = info["n"], spec["path"]
    d = _to_device(a, path)
    if info["out2"]:
        a.out2 = torch.empty(a.x.shape, dtype=spec["sd"])
        d.out2 = torch.empty(a.x.shape, dtype=spec["sd"], device="cuda")
    variant = 1 if path == "tma" else 2
    be.set_tuning(variant, 0, 0)
    try:
        gm, go = be.step(d)
    finally:
        be.set_tuning(2, 0, 0)
    with np.errstate(all="ignore"):
        wm, wo = GuidedOracle().step(a)
    what = "%s %s" % (spec, dict(param=a.param, px0=a.predict_x0, alpha=a.alpha_e, w4=a.w4, raw_round=a.raw_round,
                                 thr=None if a.thr is None else a.thr.tolist()))
    for g, w, name in ((gm, wm, "m_out"), (go, wo, "out")):
        assert (g is None) == (w is None), (name, what)
        if g is not None:
            assert_bits_equal(g, w, "%s of %s" % (name, what))
    if info["out2"]:
        assert_bits_equal(d.out2, a.out2, "out2 of " + what)
    kernels, fast_div = mirror(a, spec["md"], spec["sd"], n, path != "unaligned", variant)
    if tally is not None:
        _tally(tally, hits, spec, a, info, kernels, gm, go)
    return kernels


# ---- tallies ------------------------------------------------------------------------------------------------------
def _tally(tally, hits, spec, a, info, kernels, gm, go):
    fam, ne = spec["fam"], a.n_model
    body = kernels[0]
    lab = kernel_label(body) if a.coef_dev is None else "scalar(dev_coef)"
    fast = lab in ("direct-fast", "tma")
    for k in kernels:
        tally[(fam, kernel_label(k) if a.coef_dev is None else "scalar(dev_coef)", "launch", "")] += 1
    if ne > 0 and a.predict_x0:      # only the FAST kernels divide by alpha with the reciprocal
        tally[(fam, lab, "alpha", "recip" if fast else "ieee")] += 1
    if a.form == FORM_SS3T:
        ok = recip_div_ok(a.w4) and (not (ne > 0 and a.predict_x0) or recip_div_ok(a.alpha_e)) and a.coef_dev is None
        tally[(fam, lab, "w4", "recip" if ok else "ieee")] += 1
        if ne == 0 and body[0] == "direct" and not body[5]:
            tally[("ss3t-ne0-generic", body[2])] += 1
    if a.thr is not None:
        for s in a.thr.numpy():
            kind = "recip" if recip_div_ok(s) else ("ieee-finite" if np.isfinite(s) else "ieee-nonfinite")
            tally[(fam, lab, "thr", kind if fast else "ieee")] += 1
    if ne > 0 and a.predict_x0 and a.param == PARAM_NOISE and not fast and body[0] == "direct":
        tally[(fam, "direct-generic", "noise-network", "alpha refused" if not recip_div_ok(a.alpha_e) else "other")] += 1
    for key in ("f16 >= 65520", "f16 < 65520"):
        hits[(key,)] += info["planted"][key]
    # numerators of each division site, recomputed from the executor's operands, and the fp64 check of the quotients
    if fam != "plain" or a.state_dtype != F32 or a.raw_round:
        return
    with np.errstate(all="ignore"):
        if ne > 0 and a.predict_x0 and a.param in (PARAM_NOISE, PARAM_SCORE) and a.e_cond.dtype == F32:
            conv = (lambda v: (-f32(a.sigma_e)) * v) if a.param == PARAM_SCORE else (lambda v: v)
            eps = conv(a.e_cond.numpy().reshape(-1))
            if ne == 2:
                epu = conv(a.e_uncond.numpy().reshape(-1))
                eps = epu + f32(a.guidance) * (eps - epu)
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
            if fast and recip_div_ok(a.alpha_e):
                for t in GUARD:
                    hits[("alpha", float(t))] += int((num == t).sum())
            if a.form == FORM_NONE:
                got = gm.cpu().numpy().reshape(-1)
                fin = np.isfinite(got)
                assert (got[fin].view(np.uint32) == want[fin].view(np.uint32)).all(), \
                    ("fp64 quotient", spec, int((got[fin] != want[fin]).sum()))
                tally[("fp64 checked", "thr" if a.thr is not None else "alpha")] += int(fin.sum())
        if a.form == FORM_SS3T and recip_div_ok(a.w4) and a.coef_dev is None and \
                (ne == 0 or (a.param == PARAM_NOISE and not a.predict_x0 and a.e_cond.dtype == F32)):
            T0 = (a.m0 if ne == 0 else gm.cpu()).numpy().reshape(-1)
            m1, m2 = a.m1.numpy().reshape(-1), a.m2.numpy().reshape(-1)
            D10, D11 = f32(a.w0) * (m1 - m2), f32(a.w1) * (T0 - m2)
            n1, n2 = f32(a.w2) * D10 - f32(a.w3) * D11, f32(2) * (D11 - D10)
            for t in GUARD:
                hits[("w4", float(t))] += int((n1 == t).sum() + (n2 == t).sum())


# ---- the case list ------------------------------------------------------------------------------------------------
def _pairs(fam, ne, path):
    if ne == 0:
        return [(F32, F32)] if fam == "rnd" else [(F32, F32), (BF16, BF16), (F16, F16)]
    if fam == "rnd":
        return [(BF16, F32), (F16, F32)] + ([(F32, F32)] if path in ("direct", "unaligned") else [])
    return PAIRS + ([MIXED] if path in ("direct", "dev_coef") else [])


def case_specs():
    specs, seed = [], 0
    for fam in FAMILIES:
        for path in PATHS:
            for ne in ((0, 1, 2) if fam in ("plain", "rnd") else (2,)):
                if fam == "rnd" and path == "tma":
                    continue
                for form in range(7):
                    if form == FORM_NONE and ne == 0:
                        continue
                    for md, sd in _pairs(fam, ne, path):
                        for div in ("ok", "refused"):
                            seed += 1
                            specs.append(dict(fam=fam, path=path, ne=ne, form=form, md=md, sd=sd, div=div,
                                              seed=90000 + seed))
    return specs


REQUIRED = [("ss3t-ne0-generic", "float"), ("ss3t-ne0-generic", "__nv_bfloat16"), ("ss3t-ne0-generic", "__half"),
            ("plain", "direct-fast", "thr", "ieee-finite"), ("plain", "direct-fast", "thr", "ieee-nonfinite"),
            ("plain", "direct-fast", "thr", "recip"), ("rs", "direct-fast", "thr", "ieee-finite"),
            ("pg", "direct-fast", "thr", "ieee-finite"),
            ("plain", "direct-generic", "noise-network", "alpha refused"),
            ("plain", "direct-fast", "alpha", "recip"), ("plain", "direct-generic", "alpha", "ieee"),
            ("plain", "tma", "alpha", "recip"), ("plain", "tma", "w4", "recip"),
            ("plain", "direct-fast", "w4", "recip"), ("plain", "direct-generic", "w4", "ieee"),
            ("plain", "scalar", "w4", "recip"), ("plain", "scalar", "w4", "ieee"), ("plain", "scalar", "thr", "ieee"),
            ("plain", "scalar(dev_coef)", "w4", "ieee"), ("plain", "scalar(dev_coef)", "alpha", "ieee"),
            ("rnd", "direct-generic", "launch", ""), ("rnd", "scalar", "launch", ""),
            ("rs", "direct-fast", "launch", ""), ("rs", "direct-generic", "launch", ""), ("rs", "scalar", "launch", ""),
            ("pg", "direct-fast", "launch", ""), ("pg", "direct-generic", "launch", ""), ("pg", "scalar", "launch", ""),
            ("plain", "tma", "launch", ""), ("plain", "scalar(dev_coef)", "launch", ""),
            ("fp64 checked", "alpha"), ("fp64 checked", "thr")]
REQUIRED_HITS = ([("alpha", float(t)) for t in GUARD] + [("thr", float(t)) for t in GUARD_TINY]
                 + [("w4", float(t)) for t in GUARD] + [("f16 >= 65520",), ("f16 < 65520",)])


def test_step_kernels_at_ieee_edges(cuda_backend):
    tally, hits = Counter(), Counter()
    specs = case_specs()
    for spec in specs:
        run_case(cuda_backend, spec, tally, hits)
    print("\n%d edge-valued launches; path tally:" % len(specs))
    for k, v in sorted(tally.items(), key=str):
        print("  %-70s %d" % (k, v))
    print("numerator and boundary hits:", dict(sorted(hits.items(), key=str)))
    missing = [k for k in REQUIRED if tally[k] == 0] + [k for k in REQUIRED_HITS if hits[k] == 0]
    assert not missing, missing


def profile_mirror():
    """The dispatch mirror against torch.profiler's kernel names, one launch per kind of kernel, one profiler session
    each."""
    from dpm_solver_b200 import ops
    from torch.profiler import ProfilerActivity, profile
    be = ops.CudaBackend()
    chosen = {}
    for spec in case_specs():
        a, info = build_case(spec)
        ks, _ = mirror(a, spec["md"], spec["sd"], info["n"], spec["path"] != "unaligned",
                       1 if spec["path"] == "tma" else 2)
        key = (kernel_label(ks[0]) if a.coef_dev is None else "dev_coef", ks[0][6:9] if ks[0][0] == "direct" else (),
               spec["ne"] == 0 and spec["form"] == FORM_SS3T, len(ks))
        chosen.setdefault(key, spec)
    assert len(chosen) >= 10, chosen.keys()
    for spec in chosen.values():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ks = run_case(be, spec)
            torch.cuda.synchronize()
        ran = [e.name.replace(" ", "") for e in prof.events() if "k_step_" in e.name]
        want = [kernel_name(k) for k in ks]
        assert len(ran) == len(want) and all(w in r for w, r in zip(want, ran)), (spec, want, ran)
    print("%d profiled launches match the mirror" % len(chosen))


def test_mirror_names_the_kernel_that_ran():
    """profile_mirror() in a child process of its own, like the profiler checks of tests/test_gpu_flow.py and
    tests/test_gpu_cfg_multi_edges.py: profiler sessions opened in the test process after many others were seen to
    record no kernels, so this one neither inherits that process's profiler state nor leaves its own behind."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path[:0] = %r; import test_gpu_step_edges as t; t.profile_mirror()"
            % [root, os.path.join(root, "tests"), os.path.join(root, "tests", "golden")])
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.stdout[-4000:], r.stderr[-4000:])
    print(r.stdout.strip().splitlines()[-1])
