"""Edge-valued operands for the fused step, and the comparison rule applied to them.

The step kernels claim bit equality with the reference's eager op chain, and that claim is only as good as the data
it is checked on. This module supplies operands at the places where element-wise kernels go wrong: NaN, infinities,
signed zeros, subnormals of every storage type, values whose update overflows, fp16 results next to the
round-to-infinity boundary, numerators at the range guard of the constant division (common.cuh: div_const,
div_const8) and divisors on both sides of the host's acceptance test (recip_div_ok). Values are placed per 8-element
packet: in lane 0 (which seeds div_const8's min/max), in lane 7, in all lanes, or mixed with ordinary lanes.
"""
import math

import numpy as np
import torch

f32 = np.float32
NAN, INF = float("nan"), float("inf")


def from_bits(b):
    return np.array([b], np.uint32).view(np.float32)[0]


def nudge(v, k):
    """v moved k fp32 ulps (towards +inf for k > 0)."""
    v = f32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, f32(INF if k > 0 else -INF))
    return v


def recip_div_ok(d):
    """common.cuh recip_div_ok: |d| in [2^-20, 2^21) (biased exponent 107..147), significand not all ones."""
    b = int(np.float32(d).view(np.uint32))
    ex = (b >> 23) & 0xff
    return 107 <= ex <= 147 and (b & 0x7fffff) != 0x7fffff


# numerators at the range guard of div_const / div_const8: 1e-25 and 1e30, one ulp either side, both signs
GUARD = [s * nudge(v, k) for v in (1e-25, 1e30) for k in (-1, 0, 1) for s in (f32(1), f32(-1))]
GUARD_TINY = [g for g in GUARD if abs(g) < 1]       # the only ones a clamp to an accepted threshold lets through

# divisors (alpha_e, w4, per-sample thresholds) on both sides of recip_div_ok
DIV_OK = [f32(2.0 ** -20), nudge(2.0 ** 21, -2), from_bits(0x3F7FFFFE)]
DIV_REFUSED = [nudge(2.0 ** -20, -1), nudge(2.0 ** 21, -1), f32(2.0 ** 21), from_bits(0x3F7FFFFF)]
THR_EXTRA = [f32(0), f32(INF), f32(NAN), f32(1e-40)]
assert all(recip_div_ok(d) for d in DIV_OK) and not any(recip_div_ok(d) for d in DIV_REFUSED + THR_EXTRA)

F16_MAX, F16_INF_EDGE = 65504.0, 65520.0     # fp16: largest finite value; fp32 values from here on round to inf


def edge_pool(dtype):
    """Edge values representable in `dtype` (fp32 values rounded once to it), as fp32."""
    v = [NAN, INF, -INF, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 3e38, -3e38] + [float(g) for g in GUARD]
    if dtype == torch.bfloat16:
        v += [2.0 ** -133, -(2.0 ** -133), 2.0 ** -127, 3.0e38]           # bf16 subnormals
    elif dtype == torch.float16:
        v += [2.0 ** -24, -(2.0 ** -24), 2.0 ** -20, F16_MAX, -F16_MAX, 60000.0]   # fp16 subnormals, its largest values
    t = torch.tensor(v, dtype=torch.float32).to(dtype).float()
    return t.numpy()


PATTERNS = ("lane0", "lane7", "all", "mixed")


def lanes(pattern, rng):
    if pattern == "lane0":
        return np.array([0])
    if pattern == "lane7":
        return np.array([7])
    if pattern == "all":
        return np.arange(8)
    k = int(rng.integers(1, 8))
    return np.sort(rng.choice(8, size=k, replace=False))


def scatter_edges(streams, dtypes, rng, frac=0.4):
    """Put edge values into some packets of the fp32 arrays `streams` (name -> array of n elements, edited in place),
    one stream and one placement pattern per chosen packet. Returns the patterns used."""
    names = sorted(streams)
    n = len(streams[names[0]])
    used = []
    for pk in range(n // 8):
        if rng.random() >= frac:
            continue
        name = names[int(rng.integers(len(names)))]
        pat = PATTERNS[int(rng.integers(len(PATTERNS)))]
        idx = pk * 8 + lanes(pat, rng)
        pool = edge_pool(dtypes[name])
        streams[name][idx] = pool[rng.integers(len(pool), size=len(idx))]
        used.append(pat)
    return used


def solve(f, target, guess, reach=12):
    """An fp32 v within `reach` ulps of `guess` with f(v) == target bit for bit, or None."""
    target = f32(target)
    with np.errstate(all="ignore"):
        for k in sorted(range(-reach, reach + 1), key=abs):
            v = nudge(guess, k)
            if f32(f(v)).view(np.uint32) == target.view(np.uint32):
                return v
    return None


def bits_equal(got, want):
    """The step tests' comparison rule: NaN in the same positions, and every other element bit-identical (-0, +-inf
    and subnormals included). NaN payloads are not compared: the GPU writes canonical NaNs (fp32 0x7FFFFFFF, bf16
    0x7FFF) where torch's CPU casts write 0x7FC0. Returns (ok, description of the first mismatch)."""
    got, want = got.detach().cpu().reshape(-1), want.detach().cpu().reshape(-1)
    assert got.dtype == want.dtype, (got.dtype, want.dtype)
    gi = torch.int16 if got.element_size() == 2 else torch.int32
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    bad = (gn != wn) | (~gn & (got.view(gi) != want.view(gi)))
    if not bool(bad.any()):
        return True, ""
    i = int(bad.nonzero()[0])
    return False, "element %d: got %r (0x%x), want %r (0x%x); %d mismatches" % (
        i, float(got[i]), int(got.view(gi)[i]) & 0xffffffff, float(want[i]), int(want.view(gi)[i]) & 0xffffffff,
        int(bad.sum()))


def assert_bits_equal(got, want, what=""):
    ok, msg = bits_equal(got, want)
    assert ok, "%s: %s" % (what, msg)


def is_finite32(v):
    return math.isfinite(float(v))
