"""The exact mirror of words.cu's APG words reduction (apg_oracle.apg_words_exact), on the CPU: it is still the paper's
formula -- within an ulp of the fp64 words summed in numpy's order over many shapes and over finite edge data, with the
same non-finite results -- and its vectorised order is the kernel's, thread by thread, against a plain loop over the
CTAs, threads and lanes of the words pass."""
import numpy as np
import pytest

from apg_oracle import CHUNK, apg_final, apg_sums_exact, apg_words_exact
from test_gpu_cfg_rescale import ulp_dist

f32 = np.float32
PER_SAMPLE = [1, 7, 8, 9, 104, 1000, 8191, 8192, 8193, 8192 * 3 - 8, 16384, 3 * 8192 + 1]


def loop_sums(R, c):
    """The APG words pass and k_apg_final's merge written as plain loops (one python add per device add)."""
    Bn, ps = R.shape
    chunks = -(-ps // CHUNK)
    out = []
    for a, b in ((R, R), (R, c), (c, c)):
        tot = np.zeros(Bn)
        for s in range(Bn):
            merged = 0.0
            for ch in range(chunks):
                cnt = min(CHUNK, ps - ch * CHUNK)
                acc = [0.0] * 256
                for tid in range(256):
                    v = 0.0
                    for u in range(4):
                        for i in range(8):
                            j = (u * 256 + tid) * 8 + i
                            if j < cnt:
                                e = ch * CHUNK + j
                                v = v + float(a[s, e]) * float(b[s, e])
                    acc[tid] = v
                for o in (16, 8, 4, 2, 1):
                    acc = [acc[t] + acc[t ^ o] for t in range(256)]
                part = 0.0
                for w in range(8):
                    part = part + acc[32 * w]
                merged = merged + part
            tot[s] = merged
        out.append(tot)
    return out


@pytest.mark.parametrize("ps", [9, 104, 8193])
def test_vectorised_order_is_the_loop(ps):
    rng = np.random.default_rng(ps)
    # magnitudes spread over 2^60 so that the order of every add shows in the bits
    R = (rng.standard_normal((2, ps)) * 2.0 ** rng.integers(-30, 30, (2, ps))).astype(f32)
    c = (rng.standard_normal((2, ps)) * 2.0 ** rng.integers(-30, 30, (2, ps))).astype(f32)
    got = apg_sums_exact(R, c)
    want = loop_sums(R, c)
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()


def numpy_words(R, c, w, eta, r):
    R64, c64 = R.astype(np.float64), c.astype(np.float64)
    with np.errstate(all="ignore"):
        return apg_final((R64 * R64).sum(1), (R64 * c64).sum(1), (c64 * c64).sum(1), w, eta, r)


def regimes(rng, Bn, ps):
    """(name, R, c) fp32 [B, ps]: ordinary data and finite edges -- tiny, subnormal and huge values (squares beyond
    fp32), zeros, a sample with c = 0 or R = 0, both signs mixed per element."""
    n = rng.standard_normal
    yield "random", n((Bn, ps)), n((Bn, ps)) * 1.3 + 0.2
    yield "tiny", n((Bn, ps)) * 1e-30, n((Bn, ps)) * 1e-25
    yield "subnormal", rng.choice([1e-40, -1e-40, 1e-45, 3e-39], (Bn, ps)), n((Bn, ps)) * 1e-38
    yield "huge", n((Bn, ps)) * 1e30, n((Bn, ps)) * 3e37
    R, c = n((Bn, ps)), n((Bn, ps))
    c[0] = 0.0
    R[-1] = 0.0
    yield "zero samples", R, c
    R, c = n((Bn, ps)), n((Bn, ps))
    mask = rng.random((Bn, ps)) < 0.5
    R[mask], c[~mask] = 0.0, -0.0
    yield "sparse", R, c
    yield "wide", n((Bn, ps)) * 2.0 ** rng.integers(-60, 60, (Bn, ps)), n((Bn, ps)) * 2.0 ** rng.integers(-60, 60, (Bn, ps))


@pytest.mark.parametrize("ps", PER_SAMPLE)
def test_mirror_within_an_ulp_of_the_fp64_words(ps):
    rng = np.random.default_rng(1000 + ps)
    Bn = 3
    worst = 0
    for name, R, c in regimes(rng, Bn, ps):
        R, c = R.astype(f32), c.astype(f32)
        for eta, r, w in ((0.0, 0.0, 4.0), (0.3, 1.0, 7.5), (1.0, 1e6, -2.0), (0.5, 1e-30, 2.0)):
            wv = np.array([w, 1.0, 3.5][:Bn], np.float64)
            got = apg_words_exact(R, c, wv, eta, r)
            want = numpy_words(R, c, wv, eta, r)
            d = ulp_dist(got, want)      # (also requires the same non-finite values)
            assert d <= 1, (name, eta, r, w, d)
            worst = max(worst, d)
    assert worst <= 1


def test_nonfinite_words_follow_the_formula():
    """A NaN or an inf in a sample gives the fp64 formula's non-finite words, in that sample only."""
    rng = np.random.default_rng(3)
    R, c = rng.standard_normal((4, 9000)).astype(f32), rng.standard_normal((4, 9000)).astype(f32)
    R[0, 8500], c[1, 3], R[2, 100] = np.nan, np.inf, f32(3e38)
    w = np.full(4, 4.0)
    got = apg_words_exact(R, c, w, 0.3, 2.0)
    want = numpy_words(R, c, w, 0.3, 2.0)
    assert ulp_dist(got, want) <= 1
    assert np.isnan(got[0, 0]) and np.isnan(got[0, 1]) and np.isfinite(got[:, 3]).all()
