"""Fuzz: random forms, dtypes, sizes, pointer offsets (misalignment), aliasing and tuning against the
numpy executor, bit for bit. Seeds are fixed, the case list is not hand-picked."""
import random

import numpy as np
import pytest
import torch

from dpm_solver_b200._lib import (FORM_DIFF2, FORM_LIN1, FORM_LIN2, FORM_LIN3, FORM_MS3, FORM_NONE, FORM_SS3T,
                                  PARAM_NOISE, PARAM_SCORE, PARAM_V, PARAM_X_START)
from dpm_solver_b200.ops import StepArgs
from oracle_backend import OracleBackend

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTS = [(torch.float32, torch.float32), (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16),
       (torch.float32, torch.bfloat16), (torch.float32, torch.float16), (torch.bfloat16, torch.float16)]


def one_case(rng, be):
    form = rng.choice([FORM_NONE, FORM_LIN1, FORM_LIN2, FORM_LIN3, FORM_DIFF2, FORM_MS3, FORM_SS3T])
    n_model = rng.choice([0, 1, 2]) if form != FORM_NONE else rng.choice([1, 2])
    sdt, mdt = rng.choice(DTS)
    n = rng.choice([rng.randint(1, 64), rng.randint(65, 5000), 8 * rng.randint(100, 40000) + rng.randint(0, 7),
                    8 * 148 * 1024 + rng.randint(0, 4096)])
    off = rng.choice([0, 0, 0, 1, 3, 4, 8])                # element offset into a larger allocation
    g = torch.Generator().manual_seed(rng.randint(0, 1 << 30))
    mk = lambda dt: (torch.randn(n + 16, generator=g) * rng.choice([0.1, 1.0, 30.0])).to(dt)
    param = rng.choice([PARAM_NOISE, PARAM_NOISE, PARAM_X_START, PARAM_V, PARAM_SCORE])
    px0 = rng.random() < 0.6
    v = [rng.uniform(0.2, 1.5) * rng.choice([-1, 1]) for _ in range(9)]
    a = StepArgs(form=form, n_model=n_model, param=param, predict_x0=px0 and n_model > 0, c0_on_old=rng.random() < 0.5,
                 guidance=rng.choice([1.0, 3.5, 7.5]), alpha_e=rng.uniform(0.004, 1.0), sigma_e=rng.uniform(0.03, 1.0),
                 a=v[0], c0=v[1], c1=v[2], c2=v[3], w0=v[4], w1=v[5], w2=abs(v[6]), w3=abs(v[7]), w4=abs(v[8]) + 0.1,
                 want_m_out=rng.random() < 0.7, state_dtype=sdt)
    host, devt = {}, {}

    def put(name, dt):
        t = mk(dt)
        host[name] = t[off:off + n]
        devt[name] = t.to(DEV)[off:off + n]

    if form != FORM_NONE:
        put("x", sdt)
    if n_model == 0:
        put("m0", sdt)
    else:
        put("e_cond", mdt)
        if n_model == 2:
            put("e_uncond", mdt)
        if a.predict_x0 or param in (PARAM_X_START, PARAM_V):
            if form == FORM_NONE or rng.random() < 0.4:
                put("xe", sdt)
            else:
                host["xe"], devt["xe"] = host["x"], devt["x"]
    if form in (FORM_LIN2, FORM_LIN3, FORM_DIFF2, FORM_MS3, FORM_SS3T):
        put("m1", sdt)
    if form in (FORM_LIN3, FORM_MS3, FORM_SS3T):
        put("m2", sdt)
    ah, ad = StepArgs(**{**a.__dict__, **host}), StepArgs(**{**a.__dict__, **devt})
    if a.predict_x0 and n_model > 0 and rng.random() < 0.3 and n >= 64:
        ps = rng.choice([d for d in (8, 16, 24, 1, 7) if n % d == 0] or [n])
        thr = torch.rand(n // ps, generator=g) * 2 + 0.3
        ah.thr, ah.per_sample, ad.thr, ad.per_sample = thr, ps, thr.to(DEV), ps
    be.set_tuning(rng.choice([0, 1, 2]), rng.choice([0, 64, 128, 256, 512]), rng.choice([0, 1, 2, 4]))
    dev_coef = rng.random() < 0.25
    if dev_coef:
        # scalars in device memory (dpm_step_desc.dev_coef, CO_* layout of adaptive_ctl.cu); the by-value copies in
        # the descriptor get other values, which the launch must ignore. Division is IEEE on this path.
        names = ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4", "alpha_e", "sigma_e")
        blk = [float(np.float32(getattr(a, k) * rng.uniform(0.5, 1.5))) for k in names]
        blk[names.index("w4")] = abs(blk[names.index("w4")]) + 0.1
        ad.coef_dev = torch.tensor(blk + [0.0] * 5, dtype=torch.float32, device=DEV)
        for k, v in zip(names, blk):
            setattr(ah, k, v)
            setattr(ad, k, -3.0 * v + 0.25)
    ref_m, ref_o = OracleBackend().step(ah)
    before = be.launch_count()
    got_m, got_o = be.step(ad)
    if dev_coef:
        assert be.launch_count() - before == 1          # one generic launch reads the block
    for r, q in ((ref_m, got_m), (ref_o, got_o)):
        assert (r is None) == (q is None)
        if r is not None:
            w = torch.int16 if r.element_size() == 2 else torch.int32
            assert torch.equal(q.cpu().view(w), r.view(w)), (form, n_model, sdt, mdt, n, off, param, px0, dev_coef)


@pytest.mark.parametrize("seed", range(8))
def test_fuzz_step_kernels(cuda_backend, seed):
    rng = random.Random(4242 + seed)
    try:
        for _ in range(40):
            one_case(rng, cuda_backend)
    finally:
        cuda_backend.set_tuning(2, 0, 0)


# ---- dynamic-thresholding quantile (csrc/quantile.cu) ------------------------------------------------------------
# state dtype, network dtype: every pair of the step fuzz, the other 16-bit mix, and fp32 networks with a 16-bit state
QDTS = DTS + [(torch.float16, torch.bfloat16), (torch.bfloat16, torch.float32), (torch.float16, torch.float32)]
_CLUSTER_KEYS = 49856      # keys one CTA of the cluster kernel can park in 227 KB of shared memory (H100)


def _recip_bad(rng):
    """A divisor whose significand is all ones: recip_div_ok() refuses it, so x0 takes the IEEE division."""
    e = rng.randint(119, 126)                                     # 2^-8 .. 2^-1 (times ~2)
    return float(np.array([(e << 23) | 0x7fffff], dtype=np.uint32).view(np.float32)[0])


def _q_with_integer_pos(rng, ps):
    """A q whose fp32 rank pos = fl(q*(ps-1)) is an integer (so w = 0 and one order statistic decides)."""
    m = np.float32(ps - 1)
    for _ in range(8):
        j = rng.randint(0, ps - 1)
        q = np.float32(j) / m if m > 0 else np.float32(1)
        if float(q * m) == j:
            return float(q)
    return 1.0


def one_quantile_case(rng, be, paths):
    import os
    impl = rng.choice(["default", "default", "cluster"])
    r = rng.random()
    if r < 0.03:
        ps = rng.choice([3 * 512 * 512, 1 << 21])
    else:
        ps = rng.choice([rng.randint(1, 64), rng.randint(65, 8191), 8192 + rng.choice([-1, 0, 1, 7, 8]),
                         8 * rng.randint(1025, 1 << 15)])
    B = rng.randint(1, max(1, min(24, (1 << 21) // ps)))
    if ps > (1 << 19):
        B = rng.randint(1, max(1, (1 << 24) // ps))
    n = B * ps
    sdt, mdt = rng.choice(QDTS)
    n_model = rng.choice([1, 2])
    param = rng.choice([PARAM_NOISE, PARAM_NOISE, PARAM_X_START, PARAM_V, PARAM_SCORE])
    off = rng.choice([0, 0, 0, 1, 3, 4, 8])
    pick = lambda: rng.choice([rng.uniform(0.004, 1.0), rng.uniform(0.004, 1.0), 1.0, _recip_bad(rng)])
    alpha, sigma = pick(), pick()
    g = torch.Generator().manual_seed(rng.randint(0, 1 << 30))
    kind = rng.choice(["gauss", "gauss", "heavy", "ties"])
    scale = rng.choice([0.1, 1.0, 30.0])

    def draw(dt):
        v = torch.randn(n + 16, generator=g) * scale
        if kind == "heavy":
            v = v * torch.exp(2.0 * torch.randn(n + 16, generator=g))
        elif kind == "ties":
            v = (v * 4).round() / 4
        return v

    raw = {"xe": draw(sdt), "e_cond": draw(mdt)}
    if n_model == 2:
        raw["e_uncond"] = draw(mdt)
    # per-sample oddities: constant / all-zero samples, +-inf or NaN near the target rank, overflowing quotients
    q = rng.choice([0.0, 1.0, 0.995, 0.995, 0.5, rng.random(), _q_with_integer_pos(rng, ps)])
    lo = int(np.floor(np.float32(q) * np.float32(ps - 1)))
    special = []
    for b in range(B):
        if rng.random() > 0.3:
            continue
        what = rng.choice(["const", "zero", "inf", "nan", "overflow"])
        sl = slice(off + b * ps, off + (b + 1) * ps)
        if what in ("const", "zero"):
            c = 0.0 if what == "zero" else rng.choice([0.75, -2.5, 1e-3])
            for k in raw:
                raw[k][sl] = c if k == "xe" else 0.0
        else:
            k_bad = max(1, min(ps, ps - lo + rng.randint(-2, 1)) if what != "nan" else rng.randint(1, 3))
            idx = off + b * ps + torch.from_numpy(np.random.RandomState(b).permutation(ps)[:k_bad])
            if what == "overflow":           # finite |numerator|, |numerator / alpha| beyond the fp32 range
                if sdt == torch.float16:
                    continue
                raw["xe"][idx] = 3.0e38 * rng.choice([-1, 1])
                alpha = rng.uniform(0.004, 0.5)
            else:
                tgt = rng.choice(list(raw))
                raw[tgt][idx] = float("nan") if what == "nan" else float("inf") * rng.choice([-1, 1])
        special.append((b, what))
    host, devt = {}, {}
    for k, v in raw.items():
        t = v.to(sdt if k == "xe" else mdt)
        host[k], devt[k] = t[off:off + n], t.to(DEV)[off:off + n]
    xe_is_x = rng.random() < 0.3
    a = StepArgs(form=FORM_NONE, n_model=n_model, param=param, predict_x0=True, guidance=rng.choice([1.0, 3.5, 7.5]),
                 alpha_e=alpha, sigma_e=sigma, per_sample=ps, state_dtype=sdt)
    ah, ad = StepArgs(**a.__dict__), StepArgs(**a.__dict__)
    for d, src in ((ah, host), (ad, devt)):
        d.e_cond, d.e_uncond = src["e_cond"], src.get("e_uncond")
        if xe_is_x:
            d.x = src["xe"]                  # no separate xe: the quantile reads x
        else:
            d.xe = src["xe"]
    max_val = rng.choice([0.0, 0.1, 1.0])
    with np.errstate(all="ignore"):
        ref = OracleBackend().dynamic_threshold(ah, q, max_val).numpy()
    if impl == "cluster":
        os.environ["DPM_QUANTILE_IMPL"] = "cluster"
    try:
        got, hdr = be.dynamic_threshold(ad, q, max_val, return_stats=True)
        got = got.cpu().numpy()
    finally:
        os.environ.pop("DPM_QUANTILE_IMPL", None)
    desc = dict(impl=impl, ps=ps, B=B, sdt=sdt, mdt=mdt, n_model=n_model, param=param, off=off, alpha=alpha,
                sigma=sigma, q=q, max_val=max_val, kind=kind, scale=scale, special=special, xe_is_x=xe_is_x)
    np.testing.assert_array_equal(got, ref, err_msg=str(desc))
    fin = np.isfinite(ref)
    assert (got[fin].view(np.uint32) == ref[fin].view(np.uint32)).all(), desc
    # which implementation and path ran (mirrors launch_quantile's choice)
    mixed16 = {sdt, mdt} == {torch.bfloat16, torch.float16}
    vec = ps % 8 == 0 and off % 8 == 0 and not mixed16
    if impl == "default" and ps >= 8192:
        num_space = vec and param == PARAM_NOISE and alpha > 0
        count = "num" if num_space else ("key" if vec else "scalar")
        paths[f"pipeline count: {count}"] += 1
        for p in hdr[:, 4].tolist():
            assert p in (1, 2), desc
            paths[f"pipeline finish: path {p}"] += 1
    else:
        paths["cluster: " + ("recomputed keys" if -(-ps // 16) > _CLUSTER_KEYS else "cached keys")] += 1


def test_fuzz_dynamic_threshold(cuda_backend):
    """Seeded random quantile cases (no hand-picked list) against OracleBackend().dynamic_threshold on the same host
    tensors, bit for bit with NaN positions matching: both implementations, sample sizes on both sides of every
    threshold, every network parameterisation, CFG, all dtype pairs, misaligned views, non-finite and overflowing
    values, ties, constants, every kind of q. Then checks that each kernel path was taken."""
    from collections import Counter
    paths = Counter()
    for seed in range(8):
        rng = random.Random(5151 + seed)
        for i in range(24):
            try:
                one_quantile_case(rng, cuda_backend, paths)
            except AssertionError as e:
                raise AssertionError(f"seed {seed} case {i}: {e}") from None
    print("quantile fuzz paths:", dict(sorted(paths.items())))
    for p in ("pipeline count: num", "pipeline count: key", "pipeline count: scalar", "pipeline finish: path 1",
              "pipeline finish: path 2", "cluster: cached keys", "cluster: recomputed keys"):
        assert paths[p] > 0, (p, dict(paths))


@pytest.mark.parametrize("nbytes", [16 * 5, 16 * 4096, 16 * 7 + 2, 6, 16 * 123457 + 14, 16 * 148 * 2048 * 3 + 8])
def test_select_copy_tail(cuda_backend, nbytes):
    """k_select_copy: dst <- src byte for byte (16-byte body and the tail) when the accept word of the controller
    state is 1; dst untouched, tail included, when it is 0."""
    from helpers import product_schedule
    ctl = cuda_backend.adaptive_controller(product_schedule("sd"), torch.device(DEV), order=2, predict_x0=True, taylor=False,
                                           t_0=1e-3, theta=0.9, t_err=1e-5, discrete_input=True)
    g = torch.Generator(device=DEV).manual_seed(nbytes)
    src = torch.randint(0, 256, (nbytes + 32,), dtype=torch.uint8, device=DEV, generator=g)
    dst = torch.randint(0, 256, (nbytes + 32,), dtype=torch.uint8, device=DEV, generator=g)
    guard = dst[nbytes:].clone()
    for accept in (0, 1):
        ctl.state.view(torch.int32)[7] = accept                  # ST_ACCEPT
        before = dst.clone()
        ctl.select_copy(dst[:nbytes], src[:nbytes])
        torch.cuda.synchronize()
        assert torch.equal(dst[:nbytes], src[:nbytes] if accept else before[:nbytes]), accept
        assert torch.equal(dst[nbytes:], guard)                  # nothing past the end is written
