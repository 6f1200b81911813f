"""Edge-valued launches of the SDE and UniPC step kernels, and mirrors of their dispatch -- TEST INFRASTRUCTURE.

Importable without a GPU. `sde_specs()` / `unipc_specs()` list the seeded cases; `build_sde()` / `build_unipc()` turn a
spec into StepArgs on the host (fp32 numpy first, edges scattered by tests/step_edges.py, planted lanes, then cast to
the storage types); `plant_noise()` finishes an SDE case once its noise z is known (the lanes that depend on z: the
single-rounding pin and the fp16 round-to-infinity boundary). `sde_mirror()` and `unipc_mirror()` name the kernels a
launch runs, following capi.cu (step_sde_impl, step_unipc_impl), step_sde.cu (pick_sde, launch_step_sde),
step_unipc.cu (launch_step_unipc) and common.cuh (fast_path_ok, recip_div_ok); `sde_paths()` splits an SDE launch into
the elements its packet path and its element path serve, per noise segment (philox.cu: noise_segments)."""
import dataclasses

import numpy as np
import torch

from dpm_solver_b200._lib import (FORM_DIFF2, FORM_LIN1, FORM_MS3, PARAM_EDM, PARAM_FLOW, PARAM_NOISE, PARAM_SCORE,
                                  PARAM_V, PARAM_X_START)
from dpm_solver_b200.ops import SdeNoise, StepArgs
from sde_oracle import SdeOracle
from step_edges import (DIV_OK, DIV_REFUSED, F16_INF_EDGE, F16_MAX, GUARD, GUARD_TINY, PATTERNS, THR_EXTRA, lanes,
                        recip_div_ok, scatter_edges, solve)

f32 = np.float32
NAN, INF = float("nan"), float("inf")
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
CNAME = {F32: "float", BF16: "__nv_bfloat16", F16: "__half"}
PAIRS = [(F32, F32), (BF16, BF16), (F16, F16), (BF16, F32), (F16, F32)]     # (model, state) of the packet kernels
ELEMENT_PAIRS = [(F32, BF16), (BF16, F16), (F16, BF16), (F32, F16)]        # served by the element / scalar path only
FORMS = (FORM_LIN1, FORM_DIFF2, FORM_MS3)
KINDS = ("scalar", "per_sample", "rescale", "per_sample_rescale", "cfgzero", "tcfg")
ORDERS = [(pc, pp) for pc in range(4) for pp in range(4) if pc or pp]       # the 15 UniPC (corrector, predictor) pairs
SDE_PATHS = ("whole", "tail", "unaligned", "ragged", "zgiven")
UNIPC_PATHS = ("whole", "tail", "unaligned", "ragged", "ragged_tail")
# (samples, elements per sample) of each path; ragged_tail puts sample boundaries inside the scalar tail
SHAPES = {"whole": (4, 64), "zgiven": (4, 64), "unaligned": (4, 64), "tail": (3, 67), "ragged": (6, 12)}
RAGGED_TAIL = [(7, 3), (6, 5)]
ORDINARY = [0.9, -0.3, 0.2, 0.1, 1.5, 0.7, 0.4, 0.6, -1.1]
THRESHOLDS = DIV_OK + DIV_REFUSED + THR_EXTRA + [f32(1.3), f32(0.6), f32(2.5)]   # as tests/test_gpu_step_edges.py
WORDS = [0.0, -0.0, 1.0, NAN, INF, -INF, 1e-40, 0.8, 1.7]      # ratios, s*, TCFG words
SCALES = WORDS + [3.5, 7.5]                                   # per-sample guidance scales
CZ = [0.0, -0.0, 1e-40, 3e38, 0.37]
PIN_CZ = 0.37
SEGMENT_MAX = 1 << 29     # philox.cu fits_32bit_indexing: an fp32 draw of more elements is split in halves


class GivenNoise(SdeOracle):
    """SdeOracle whose draw is a given z (fp32, storage order) in place of its generator's."""

    def __init__(self, z):
        super().__init__()
        self.z = z

    def draw(self, a):
        return self.z.reshape(a.x.shape).clone()


def _pick(rng, seq):
    return seq[int(rng.integers(len(seq)))]


def _grid(dtype, lo=0.0, hi=INF):
    """Every finite value of a 16-bit `dtype` with lo <= |v| < hi, both signs, as fp32."""
    bits = torch.arange(0, 0x7f80 if dtype == BF16 else 0x7c00, dtype=torch.int32).to(torch.int16)
    g = bits.view(dtype).float().numpy()
    g = g[(np.abs(g) >= lo) & (np.abs(g) < hi)]
    return np.concatenate([g, -g])


def _round16(v, dtype):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(v, dtype=f32))).to(dtype).float().numpy()


def _bits16(v, dtype):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(v, dtype=f32))).to(dtype).view(torch.int16).numpy()


# ---- the case lists ---------------------------------------------------------------------------------------------
def sde_specs():
    specs, seed = [], 0
    for ne in (0, 1, 2):
        for kind in (KINDS if ne == 2 else (None,)):
            for path in SDE_PATHS:
                for div in (("ok", "refused") if ne else ("ok",)):
                    for form in FORMS:
                        pairs = [(s, s) for s in (F32, BF16, F16)] if ne == 0 else PAIRS + ELEMENT_PAIRS[:2]
                        if ne == 2 and path not in ("whole", "zgiven"):
                            pairs = pairs[form::3]          # (every pair over the three forms)
                        for md, sd in pairs:
                            seed += 1
                            specs.append(dict(fam="sde", ne=ne, kind=kind, path=path, div=div, form=form, md=md,
                                              sd=sd, seed=51000 + seed))
    return specs


def unipc_specs():
    specs, seed = [], 0
    for ne in (0, 1, 2):
        for path in UNIPC_PATHS:
            for div in (("ok", "refused") if ne else ("ok",)):
                pairs = [(s, s) for s in (F32, BF16, F16)] if ne == 0 else PAIRS + ELEMENT_PAIRS[:2]
                for k, (pc, pp) in enumerate(ORDERS):
                    if ne == 2 and path not in ("whole",) and k % 3:
                        continue
                    for md, sd in pairs:
                        seed += 1
                        specs.append(dict(fam="unipc", ne=ne, path=path, div=div, pc=pc, pp=pp, md=md, sd=sd,
                                          seed=71000 + seed))
    return specs


# ---- building one case ------------------------------------------------------------------------------------------
def _shape(spec, rng):
    if spec["path"] == "ragged_tail":
        return RAGGED_TAIL[int(rng.integers(len(RAGGED_TAIL)))]
    return SHAPES[spec["path"]]


def _common(spec, rng, with_xe):
    """The model stage of a case: parameterisation, divisors, thresholds, streams (fp32 numpy, edges scattered later).
    with_xe: the network input may be a stream of its own (dpm_step_unipc evaluates the conversion at x)."""
    ne, md, sd = spec["ne"], spec["md"], spec["sd"]
    B, ps = _shape(spec, rng)
    n = B * ps
    refused = spec["div"] == "refused"
    if ne == 0:
        param, px0 = PARAM_NOISE, False
    else:
        param = PARAM_NOISE if (refused and rng.random() < 0.7) or rng.random() < 0.5 else \
            _pick(rng, [PARAM_X_START, PARAM_V, PARAM_SCORE, PARAM_FLOW, PARAM_EDM])
        px0 = refused or rng.random() < 0.7 or spec["path"] in ("ragged", "ragged_tail")
    alpha = _pick(rng, DIV_REFUSED) if refused else _pick(rng, DIV_OK + [f32(0.8), f32(0.6)])
    a = StepArgs(n_model=ne, param=param, predict_x0=px0, guidance=float(_pick(rng, [1.0, 3.5, 7.5])),
                 alpha_e=float(alpha), sigma_e=float(_pick(rng, [0.6, 0.03, 1.0])), want_m_out=ne > 0,
                 state_dtype=sd, per_sample=ps)
    streams, dtypes = {}, {}

    def add(name, dt, scale=1.0):
        streams[name] = (rng.standard_normal(n) * scale).astype(f32)
        dtypes[name] = dt
    add("x", sd)
    if ne == 0:
        add("m0", sd)
    else:
        add("e_cond", md, 1.3)
        if ne == 2:
            add("e_uncond", md)
        if with_xe and rng.random() < 0.4:
            add("xe", sd)
    thr = None
    if ne > 0 and px0 and (spec["path"] in ("ragged", "ragged_tail") or rng.random() < 0.6):
        thr = np.array([_pick(rng, THRESHOLDS) for _ in range(B)], dtype=f32)
    return a, streams, dtypes, thr, dict(n=n, B=B, ps=ps, pin=[], f16=[])


def _plant_model(spec, rng, a, streams, thr, info, plain):
    """x0 numerators at GUARD (eps = 0, so num = xe) and clamp numerators at GUARD_TINY in a sample whose threshold
    is accepted, in fp32 launches whose model stage is the plain combine."""
    n, ps, B = info["n"], info["ps"], info["B"]
    if not (plain and spec["sd"] == F32 and spec["md"] == F32 and a.n_model > 0 and a.predict_x0
            and a.param in (PARAM_NOISE, PARAM_SCORE)):
        return
    xe_name = "xe" if "xe" in streams else "x"
    npk = n // 8

    def packets(k):
        return [(pk, lanes(_pick(rng, PATTERNS), rng)) for pk in rng.choice(npk, size=min(k, npk), replace=False)]

    def zero_eps(i):
        for s in ("e_cond", "e_uncond"):
            if s in streams:
                streams[s][i] = 0.0
    for pk, ls in packets(3):
        for l in ls:
            i = pk * 8 + l
            zero_eps(i)
            streams[xe_name][i] = GUARD[i % len(GUARD)]
    if thr is not None:
        b = int(rng.integers(B))
        thr[b] = _pick(rng, DIV_OK + [f32(1.3)])
        alpha = f32(a.alpha_e)
        for pk, ls in packets(3 * B):
            for l in ls:
                i = pk * 8 + l
                if i // ps != b:
                    continue
                t = GUARD_TINY[i % len(GUARD_TINY)]
                xe = solve(lambda v: v / alpha, t, f32(t * alpha))
                if xe is not None:
                    zero_eps(i)
                    streams[xe_name][i] = xe


def _finish(a, streams, dtypes, thr, info, spec):
    B, ps = info["B"], info["ps"]
    for k, v in streams.items():
        setattr(a, k, torch.from_numpy(v).to(dtypes[k]).reshape(B, ps))
    if a.n_model > 0 and a.xe is None:
        a.xe = a.x
    if thr is not None:
        a.thr = torch.from_numpy(thr)
    return a, info


def build_sde(spec):
    """Host StepArgs (a.sde set, its generator left for the caller) of one SDE case, and what the checks need."""
    rng = np.random.default_rng(spec["seed"])
    a, streams, dtypes, thr, info = _common(spec, rng, True)
    ne, form, sd, kind = spec["ne"], spec["form"], spec["sd"], spec["kind"]
    a.form = form
    for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3"):
        setattr(a, k, float(f32(_pick(rng, ORDINARY))))
    if form in (FORM_DIFF2, FORM_MS3):
        streams["m1"], dtypes["m1"] = rng.standard_normal(info["n"]).astype(f32), sd
    if form == FORM_MS3:
        streams["m2"], dtypes["m2"] = rng.standard_normal(info["n"]).astype(f32), sd
    scatter_edges(streams, dtypes, rng)
    # lanes planted once z is known: the single-rounding pin (16-bit state) and the fp16 boundary of o + cz*z
    pinnable = ne == 0 and form == FORM_LIN1 and sd != F32 and spec["path"] in ("whole", "tail", "zgiven")
    cz = PIN_CZ if pinnable and rng.random() < 0.7 else _pick(rng, CZ)
    if pinnable and cz == PIN_CZ:
        a.a, a.c0 = 0.9, 0.6
        npk = info["n"] // 8
        chosen = rng.choice(npk, size=min(6, npk), replace=False)
        info["pin"] = [int(pk) * 8 + int(l) for pk in chosen[:3] for l in lanes(_pick(rng, PATTERNS), rng)]
        if sd == F16:
            info["f16"] = [(int(pk) * 8 + int(l), bool(rng.random() < 0.5))
                           for pk in chosen[3:] for l in lanes(_pick(rng, PATTERNS), rng)]
    _plant_model(spec, rng, a, streams, thr, info, kind in (None, "scalar"))
    a, info = _finish(a, streams, dtypes, thr, info, spec)
    B = info["B"]

    def words(k, pool):
        return torch.tensor([_pick(rng, pool) for _ in range(B * k)], dtype=torch.float32).reshape((B, k) if k > 1
                                                                                                    else (B,))
    if kind in ("per_sample", "per_sample_rescale") or (kind in ("cfgzero", "tcfg") and rng.random() < 0.5):
        a.guidance_b = words(1, SCALES)
    if kind in ("rescale", "per_sample_rescale"):
        a.ratio, a.phi = words(1, WORDS), float(_pick(rng, [0.7, 0.0]))
    if kind == "cfgzero":
        a.cfgzero_s = words(1, WORDS)
    if kind == "tcfg":
        a.tcfg_w = words(2, WORDS)
    a.sde = SdeNoise(float(cz))
    if rng.random() < 0.3:
        a.out2 = torch.empty(B, info["ps"], dtype=sd)
    return a, info


def plant_noise(a, info, z):
    """The lanes of an SDE case that depend on its noise z (fp32 numpy, storage order): x chosen on the 16-bit grid so
    that fl(fl32(o) + cz*z) and fl(fl(o) + cz*z) differ (o = a*x + c0*m0), and fp16 results o + cz*z on both sides of
    65520. Edits a.x / a.m0 in place; records what it planted in info."""
    if not info["pin"] and not info["f16"]:
        return
    sd = a.state_dtype
    x, m0 = a.x.float().numpy().reshape(-1).copy(), a.m0.float().numpy().reshape(-1).copy()
    A, c0, cz = f32(a.a), f32(a.c0), f32(a.sde.cz)
    rng = np.random.default_rng(len(x) + len(info["pin"]))
    cand = _grid(sd, 0.25, 64.0)
    info["pinned"] = []
    with np.errstate(all="ignore"):
        for i in info["pin"]:
            m0[i] = _round16(rng.standard_normal(), sd)
            o = A * cand + c0 * m0[i]
            once = _bits16(o + cz * z[i], sd)
            twice = _bits16(_round16(o, sd) + cz * z[i], sd)
            hit = np.nonzero(once != twice)[0]
            if len(hit):
                x[i] = cand[hit[int(rng.integers(len(hit)))]]
                info["pinned"].append(i)
        full = _grid(F16)
        info["f16_sides"] = []
        for i, side in info["f16"]:
            for free in ("x", "m0"):     # one operand at +-65504, the other searched over every finite fp16
                fixed = f32(np.sign(A if free == "m0" else c0) * F16_MAX)
                r = ((A * fixed + c0 * full) if free == "m0" else (A * full + c0 * fixed)) + cz * z[i]
                ok = (r >= F16_INF_EDGE) if side else (r < F16_INF_EDGE) & (r > 60000)
                if not ok.any():
                    continue
                j = np.nonzero(ok)[0][np.argmin(r[ok])] if side else np.nonzero(ok)[0][np.argmax(r[ok])]
                (m0 if free == "m0" else x)[i] = full[j]
                (x if free == "m0" else m0)[i] = fixed
                info["f16_sides"].append(side)
                break
    a.x = torch.from_numpy(x).to(sd).reshape(a.x.shape)
    a.m0 = torch.from_numpy(m0).to(sd).reshape(a.m0.shape)


def _uni_words(rng, pc, pp):
    from dpm_solver_b200 import plan as P
    u = lambda lo, hi: float(f32(rng.uniform(lo, hi)))
    return P.UniCoeffs(pc, pp, (u(-1, 1), u(-1, 1)), u(-1, 1), u(0.5, 1.5), u(-1, 1), (u(-1, 1), u(-1, 1)))


def build_unipc(spec):
    """Host StepArgs (a.unipc set) of one UniPC case, and what the checks need."""
    rng = np.random.default_rng(spec["seed"])
    a, streams, dtypes, thr, info = _common(spec, rng, False)
    ne, sd, pc, pp = spec["ne"], spec["sd"], spec["pc"], spec["pp"]
    a.form = FORM_LIN1
    w = _uni_words(rng, pc, pp)
    a.unipc = w
    n = info["n"]
    for k in ("m1", "m2", "m3"):
        streams[k], dtypes[k] = rng.standard_normal(n).astype(f32), sd
    scatter_edges(streams, dtypes, rng)
    # fp16 state: the corrected state c (m_{i-1..i-3} = 0, so c = x + ct*m0) and the predictor output (m_{i-1..i-3} =
    # m0, so c = x and o = a*x + c0*m0) on both sides of 65520
    if sd == F16 and ne == 0:
        full = _grid(F16)
        npk = n // 8
        for pk in rng.choice(npk, size=min(3, npk), replace=False):
            for l in lanes(_pick(rng, PATTERNS), rng):
                i = int(pk) * 8 + int(l)
                side = bool(rng.random() < 0.5)
                what = "c" if pc > 0 and (pp == 0 or rng.random() < 0.5) else "out"
                k0 = f32(w.ct) if what == "c" else f32(w.c0)
                fixed = f32(np.sign(k0) * F16_MAX) if k0 != 0 else f32(F16_MAX)
                with np.errstate(all="ignore"):
                    r = full + k0 * fixed if what == "c" else f32(w.a) * full + k0 * fixed
                ok = (r >= F16_INF_EDGE) if side else (r < F16_INF_EDGE) & (r > 60000)
                if not ok.any():
                    continue
                idx = np.nonzero(ok)[0]
                j = idx[np.argmin(r[ok])] if side else idx[np.argmax(r[ok])]
                streams["x"][i], streams["m0"][i] = full[j], fixed
                for k in ("m1", "m2", "m3"):
                    streams[k][i] = 0.0 if what == "c" else fixed
                info["f16"].append((what, side))
    _plant_model(spec, rng, a, streams, thr, info, True)
    a, info = _finish(a, streams, dtypes, thr, info, spec)
    a.m3 = a.m3 if pc == 3 else None
    B, ps = info["B"], info["ps"]
    if pp > 0 and rng.random() < 0.3:
        a.out2 = torch.empty(B, ps, dtype=sd)
    if pp == 0 or rng.random() < 0.5:
        a.out_c = torch.empty(B, ps, dtype=sd)
    return a, info


def to_device(a, path):
    """The device StepArgs of host args `a`: every stream one element into a larger buffer for the unaligned path, x a
    strided view for the given-z path (the launch then runs on row-major copies with torch's draw of z), outputs
    fresh."""
    d = dataclasses.replace(a)
    for f in ("x", "xe", "m0", "m1", "m2", "m3", "e_cond", "e_uncond"):
        t = getattr(a, f)
        if t is None or (f == "xe" and t is a.x):
            continue
        t = t.cuda()
        if path == "unaligned":
            buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
            buf[1:].copy_(t.reshape(-1))
            t = buf[1:].view(t.shape)
        elif path == "zgiven" and f == "x":
            buf = torch.empty(t.shape[0], 2 * t.shape[1], dtype=t.dtype, device="cuda")
            buf[:, ::2].copy_(t)
            t = buf[:, ::2]
        setattr(d, f, t)
    if a.xe is not None and a.xe is a.x:
        d.xe = d.x
    for f in ("thr", "ratio", "guidance_b", "cfgzero_s", "tcfg_w"):
        if getattr(a, f) is not None:
            setattr(d, f, getattr(a, f).cuda())
    for f in ("out2", "out_c"):
        if getattr(a, f) is not None:
            setattr(d, f, torch.empty(getattr(a, f).shape, dtype=getattr(a, f).dtype, device="cuda"))
    return d


# ---- the dispatch, mirrored -------------------------------------------------------------------------------------
def fast_div(a):
    """capi.cu build_params: every divisor the launch touches passes recip_div_ok (alpha_e of a dividing x0 step)."""
    need_alpha = a.n_model >= 1 and a.predict_x0 and a.param not in (PARAM_FLOW, PARAM_EDM)
    return not need_alpha or recip_div_ok(f32(a.alpha_e))


def fast_path_ok(a):
    """common.cuh fast_path_ok of a LIN1 / DIFF2 / MS3 launch."""
    if a.n_model == 0:
        return True
    if a.param not in (PARAM_NOISE, PARAM_FLOW, PARAM_EDM):
        return False
    if a.param == PARAM_NOISE and a.predict_x0 and not fast_div(a):
        return False
    pkps = a.per_sample // 8 if a.per_sample % 8 == 0 else 0
    if (a.thr is not None or a.ratio is not None or a.guidance_b is not None) and pkps == 0:
        return False
    return True


def _pair(a, md):
    te = a.state_dtype if a.n_model == 0 else md
    return te, (te, a.state_dtype) in PAIRS and (a.n_model > 0 or te == a.state_dtype)


def sde_mirror(a, md):
    """(kernel, vec) of an SDE launch: kernel = ("sde", TE, TS, NE, FORM, FAST, GK) as pick_sde and launch_step_sde
    choose it (the element-only <float, float, 0, LIN1, true, 0> for other dtype pairs); vec = the packet path may
    serve whole packets (before the per-segment base test). `aligned` and `z_given` describe the device operands."""
    zt = a.cfgzero_s is not None or a.tcfg_w is not None
    guided = a.guidance_b is not None or zt
    rs = a.ratio is not None and not guided
    fast = fast_path_ok(a) and not zt
    te, pair_ok = _pair(a, md)
    if not pair_ok:
        return ("sde", F32, F32, 0, FORM_LIN1, True, 0)
    ne = a.n_model
    gk = 0 if ne < 2 else (2 if guided else (1 if rs else 0))
    return ("sde", te, a.state_dtype, ne, a.form, True if ne == 0 else fast, gk)


def noise_segments(n):
    """philox.cu noise_segments: [(base, len)] of ATen's launches of an fp32 draw of n elements."""
    if n <= SEGMENT_MAX:
        return [(0, n)]
    out = []

    def split(base, ln):
        if ln > SEGMENT_MAX:
            split(base, ln // 2)
            split(base + ln // 2, ln - ln // 2)
        else:
            out.append((base, ln))
    split(0, n)
    return out


def sde_paths(a, md, n, aligned, z_given):
    """[(base, len, packet elements, element elements)] per noise segment of an SDE launch (launch_step_sde and
    k_step_sde: a segment's packets take sde_packet when vec holds and its base is a multiple of 8, a packet that
    crosses the segment's end takes sde_element)."""
    kern = sde_mirror(a, md)
    _, pair_ok = _pair(a, md)
    words = any(getattr(a, f) is not None for f in ("thr", "ratio", "guidance_b", "cfgzero_s", "tcfg_w"))
    pkps = a.per_sample // 8 if a.per_sample % 8 == 0 else 0
    vec = pair_ok and aligned and not (words and pkps == 0)
    segs = [(0, n)] if z_given else noise_segments(n)
    out = []
    for base, ln in segs:
        pk = (ln // 8) * 8 if vec and base % 8 == 0 else 0
        out.append((base, ln, pk, ln - pk))
    return kern, out


def unipc_mirror(a, md, n, aligned):
    """The kernels of a UniPC launch, as ("unipc", TE, TS, NE, FAST) and ("unipc_scalar",), following step_unipc_impl
    and launch_step_unipc."""
    te, pair_ok = _pair(a, md)
    body = ("unipc", te, a.state_dtype, a.n_model, True if a.n_model == 0 else fast_path_ok(a)) if pair_ok else None
    if n // 8 > 0 and aligned and body is not None:
        return [body] + ([("unipc_scalar",)] if n % 8 else [])
    return [("unipc_scalar",)]


def kernel_name(k):
    """The leading template arguments of the kernel's demangled name."""
    b = lambda v: "true" if v else "false"
    if k[0] == "sde":
        return "k_step_sde<%s,%s,%d,%d,%s,%d>" % (CNAME[k[1]], CNAME[k[2]], k[3], k[4], b(k[5]), k[6])
    if k[0] == "unipc":
        return "k_step_unipc<%s,%s,%d,%s>" % (CNAME[k[1]], CNAME[k[2]], k[3], b(k[4]))
    return "k_step_unipc_scalar"


# ---- tallies ------------------------------------------------------------------------------------------------------
def thr_kind(s):
    return "recip" if recip_div_ok(s) else ("ieee-finite" if np.isfinite(s) else "ieee-nonfinite")


def tally_launch(tally, spec, a, info):
    """Count one launch under (family, kernel, division site, recip / ieee, path) keys, from the mirror alone."""
    fam, md = spec["fam"], spec["md"]
    n = info["n"]
    aligned = spec["path"] != "unaligned"
    runs = []      # (kernel label, path, elements)
    if fam == "sde":
        kern, segs = sde_paths(a, md, n, aligned, spec["path"] == "zgiven")
        lab = "fast" if kern[5] else "generic"
        for _, _, pk, el in segs:
            if pk:
                runs.append((lab, "packet"))
            if el:
                runs.append(("element", "element"))
    else:
        for k in unipc_mirror(a, md, n, aligned):
            runs.append((("fast" if k[4] else "generic"), "packet") if k[0] == "unipc" else ("scalar", "scalar"))
    for lab, path in set(runs):
        tally[(fam, lab, path, "launch", "")] += 1
        fast = lab == "fast"
        if a.n_model > 0 and a.predict_x0 and a.param not in (PARAM_FLOW, PARAM_EDM):
            tally[(fam, lab, path, "alpha", "recip" if fast else "ieee")] += 1
            if a.param == PARAM_NOISE and not fast and not recip_div_ok(f32(a.alpha_e)):
                tally[(fam, lab, path, "noise-network", "alpha refused")] += 1
        if a.thr is not None:
            for s in a.thr.numpy():
                tally[(fam, lab, path, "thr", thr_kind(s) if fast else "ieee")] += 1
        if fam == "sde" and (a.cfgzero_s is not None or a.tcfg_w is not None):
            tally[(fam, lab, path, "cfgzero" if a.cfgzero_s is not None else "tcfg", "")] += 1
    return runs


def guard_hits(hits, spec, a, info, runs):
    """Numerators at the division guard in lanes a FAST packet kernel divides with the reciprocal, recomputed from the
    executor's operands: x0 numerators at GUARD (alpha) and clamp numerators at GUARD_TINY (accepted thresholds)."""
    if ("fast", "packet") not in runs or a.n_model == 0 or not a.predict_x0 \
            or a.param not in (PARAM_NOISE, PARAM_SCORE):
        return
    if a.state_dtype != F32 or a.e_cond.dtype != F32 or not recip_div_ok(f32(a.alpha_e)):
        return
    if any(getattr(a, f) is not None for f in ("ratio", "guidance_b", "cfgzero_s", "tcfg_w")):
        return
    fam = spec["fam"]
    npk8 = (info["n"] // 8) * 8
    with np.errstate(all="ignore"):
        conv = (lambda v: (-f32(a.sigma_e)) * v) if a.param == PARAM_SCORE else (lambda v: v)
        eps = conv(a.e_cond.numpy().reshape(-1))
        if a.n_model == 2:
            epu = conv(a.e_uncond.numpy().reshape(-1))
            eps = epu + f32(a.guidance) * (eps - epu)
        xe = a.xe.numpy().reshape(-1)
        num = (xe - f32(a.sigma_e) * eps)[:npk8]
        for t in GUARD:
            hits[(fam, "alpha", float(t))] += int((num == t).sum())
        if a.thr is not None:
            x0 = (num.astype(np.float64) / np.float64(f32(a.alpha_e))).astype(f32)
            s = np.repeat(a.thr.numpy(), a.per_sample)[:npk8]
            c = np.where(x0 > s, s, np.where(x0 < -s, -s, x0))
            acc = np.array([recip_div_ok(v) for v in s])
            for t in GUARD_TINY:
                hits[(fam, "thr", float(t))] += int(((c == t) & acc).sum())


def required():
    """The (family, kernel, path, site, kind) keys every run of the case lists must reach."""
    keys = []
    for fam, pk, el in (("sde", "packet", ("element", "element")), ("unipc", "packet", ("scalar", "scalar"))):
        keys += [(fam, "fast", pk, "alpha", "recip"), (fam, "generic", pk, "alpha", "ieee"),
                 (fam, "generic", pk, "noise-network", "alpha refused"),
                 (fam, "fast", pk, "thr", "recip"), (fam, "fast", pk, "thr", "ieee-finite"),
                 (fam, "fast", pk, "thr", "ieee-nonfinite"), (fam, "generic", pk, "thr", "ieee"),
                 (fam, "fast", pk, "launch", ""), (fam, "generic", pk, "launch", ""), (fam,) + el + ("launch", ""),
                 (fam,) + el + ("alpha", "ieee"), (fam,) + el + ("thr", "ieee")]
    keys += [("sde", "generic", "packet", "cfgzero", ""), ("sde", "generic", "packet", "tcfg", ""),
             ("sde", "element", "element", "cfgzero", ""), ("sde", "element", "element", "tcfg", "")]
    return keys


def required_hits():
    out = []
    for fam in ("sde", "unipc"):
        out += [(fam, "alpha", float(t)) for t in GUARD] + [(fam, "thr", float(t)) for t in GUARD_TINY]
    out += [("sde", "f16 >= 65520"), ("sde", "f16 < 65520"), ("sde", "rounding pin")]
    out += [("unipc", w, s) for w in ("c", "out") for s in ("f16 >= 65520", "f16 < 65520")]
    return out


def planted_hits(hits, spec, info):
    if spec["fam"] == "sde":
        hits[("sde", "rounding pin")] += len(info.get("pinned", []))
        for side in info.get("f16_sides", []):
            hits[("sde", "f16 >= 65520" if side else "f16 < 65520")] += 1
    else:
        for what, side in info["f16"]:
            hits[("unipc", what, "f16 >= 65520" if side else "f16 < 65520")] += 1
