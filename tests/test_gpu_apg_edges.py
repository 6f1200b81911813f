"""Adaptive projected guidance on the H100 at IEEE edges: NaN, infinities, signed zeros, subnormals and values whose
guidance difference overflows, scattered (step_edges.scatter_edges) into one sample's x, conditional and unconditional
outputs and momentum buffer, for every parameterisation and dtype pair, on the vector words path with the direct step
kernel and on the element-wise words path with k_step_scalar_apg. The words, R and the step's outputs must equal the
exact oracle bit for bit, and every other sample must come out as in a run where the edge sample is finite (words.cu:
the words of sample b depend on its values only). Built cases: c = 0 in one sample, out_c == out_u (R = 0 with a
threshold), R beyond fp32, one NaN, an infinite R on a bypassed row (its output is c exactly) and the smallest positive
threshold; where the fp64 formula (APG64) defines the result, the non-finite pattern is its pattern."""
import numpy as np
import pytest
import torch

from apg_oracle import APG64, APGOracle
from step_edges import assert_bits_equal, scatter_edges
from test_apg import W
from test_gpu_apg import COEF, DT, PAIRS, cpu
from test_gpu_apg_exact import unaligned

pytestmark = pytest.mark.gpu
Bn, EDGE = 3, 1          # three samples, the edges in sample 1


def rounded(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(dt).float().numpy()


def finite_arrays(pair, ps, rng):
    md, sd = DT[pair[0]], DT[pair[1]]
    n = rng.standard_normal
    return {"xe": rounded(n((Bn, ps)), sd), "ec": rounded(n((Bn, ps)) * 1.3 + 0.2, md), "eu": rounded(n((Bn, ps)), md),
            "rp": n((Bn, ps)).astype(np.float32)}


def run(be, pair, param, px0, form, arr, path, beta, eta, r, scales=None):
    """Words, R and the step of one launch on the device -> (words, R or None, m_out, out or None, StepArgs)."""
    from dpm_solver_b200.ops import StepArgs
    md, sd = DT[pair[0]], DT[pair[1]]
    ps = arr["xe"].shape[1]
    x = torch.from_numpy(arr["xe"]).to(sd).cuda()
    eu = torch.from_numpy(arr["eu"]).to(md).cuda()
    al, sg = (0.8, 0.6) if param != 5 else (0.2, 0.45)
    a = StepArgs(form=form, n_model=2, x=x if form else None, xe=x, e_cond=torch.from_numpy(arr["ec"]).to(md).cuda(),
                 e_uncond=unaligned(eu) if path == "element-wise" else eu, param=param, predict_x0=px0, guidance=W,
                 alpha_e=al, sigma_e=sg, alpha_t=0.8, sigma_t=0.6, state_dtype=sd, want_m_out=True, per_sample=ps, **COEF)
    if scales is not None:
        a.guidance_b = torch.tensor(scales, dtype=torch.float32).cuda()
    r_prev = torch.from_numpy(arr["rp"]).cuda() if beta else None
    r_out = torch.empty(Bn, ps, device="cuda") if beta else None
    a.apg_words = be.apg_words(a, eta, r, beta, r_prev, r_out)
    a.apg_r = r_out
    m, o = be.step(a)
    return a.apg_words, r_out, m, o, a, r_prev


def check_vs_oracle(res, eta, r, beta, what):
    words, r_out, m, o, a, r_prev = res
    ro = torch.empty(r_out.shape) if beta else None
    c = cpu(a)
    want = APGOracle(exact=True).apg_words(c, eta, r, beta, None if r_prev is None else r_prev.cpu(), ro)
    assert_bits_equal(words, want, what + ": words")
    if beta:
        assert_bits_equal(r_out, ro, what + ": R")
    c.apg_words, c.apg_r = want, ro
    mw, ow = APGOracle(exact=True).step(c)
    assert_bits_equal(m, mw, what + ": model value")
    if ow is not None:
        assert_bits_equal(o, ow, what + ": update")


def check_isolated(res, ref, beta, what):
    """Samples other than EDGE: the bits of the run with finite data in EDGE."""
    keep = [b for b in range(Bn) if b != EDGE]
    assert_bits_equal(res[0][:, keep], ref[0][:, keep], what + ": other samples' words")
    for i, name in ((1, "R"), (2, "model value"), (3, "update")):
        if res[i] is not None:
            assert_bits_equal(res[i][keep], ref[i][keep], what + ": other samples' " + name)


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("path", ["vector", "element-wise"])
@pytest.mark.parametrize("ps", [104, 8192 + 16])
def test_scattered_edges(cuda_backend, pair, path, ps):
    rng = np.random.default_rng(ps + 7 * PAIRS.index(pair) + (path == "vector"))
    md, sd = DT[pair[0]], DT[pair[1]]
    dtypes = {"xe": sd, "ec": md, "eu": md, "rp": torch.float32}
    for param in range(6):
        for rep, (eta, r, beta, px0, form) in enumerate(((0.3, 2.0, -0.5, True, 0), (0.0, 0.0, 0.3, False, 1),
                                                         (1.0, 1e6, 0.0, True, 1))):
            fin = finite_arrays(pair, ps, rng)
            arr = {k: v.copy() for k, v in fin.items()}
            names = ("xe", "ec", "eu", "rp") if beta else ("xe", "ec", "eu")
            scatter_edges({k: arr[k][EDGE].reshape(-1) for k in names}, dtypes, rng, frac=0.3)
            scales = [W, W, -2.0] if rep == 1 else None
            what = "%s param %d eta %g r %g beta %g predict_x0 %s form %d" % (path, param, eta, r, beta, px0, form)
            res = run(cuda_backend, pair, param, px0, form, arr, path, beta, eta, r, scales)
            check_vs_oracle(res, eta, r, beta, what)
            check_isolated(res, run(cuda_backend, pair, param, px0, form, fin, path, beta, eta, r, scales), beta, what)


# ---- built cases -----------------------------------------------------------------------------------------------------

def fp64_guided(res, eta, r, scales=None):
    """APG64 on the step's c and u (fp32, widened) of the launch `res` -> [B, ...] float64."""
    a = cpu(res[4])
    o = APGOracle()
    xe = a.xe.float().numpy()
    c = o._x0(a, a.e_cond.float().numpy(), xe)
    u = o._x0(a, a.e_uncond.float().numpy(), xe)
    w = np.full(Bn, W) if scales is None else np.array(scales)
    with np.errstate(all="ignore"):
        return APG64(eta, r)(c, u, w), c


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("path", ["vector", "element-wise"])
@pytest.mark.parametrize("param", range(6))
def test_built_edges(cuda_backend, pair, path, param):
    ps = 8192 + 16
    rng = np.random.default_rng(param)
    md = DT[pair[0]]

    def case(edit, eta=0.3, r=2.0, beta=0.0, scales=None, px0=True, form=0):
        fin = finite_arrays(pair, ps, rng)
        arr = {k: v.copy() for k, v in fin.items()}
        edit(arr)
        res = run(cuda_backend, pair, param, px0, form, arr, path, beta, eta, r, scales)
        what = "%s param %d: %s" % (path, param, edit.__doc__)
        check_vs_oracle(res, eta, r, beta, what)
        check_isolated(res, run(cuda_backend, pair, param, px0, form, fin, path, beta, eta, r, scales), beta, what)
        return res, what

    def c_zero(arr):
        """c = 0 in one sample"""
        arr["xe"][EDGE], arr["ec"][EDGE] = 0.0, 0.0
    res, what = case(c_zero)
    g64, c = fp64_guided(res, 0.3, 2.0)
    assert np.isfinite(g64).all() and torch.isfinite(res[2].float()).all(), what

    def d_zero(arr):
        """out_c == out_u: R = 0 with r > 0"""
        arr["eu"][EDGE] = arr["ec"][EDGE]
    res, what = case(d_zero)
    g64, c = fp64_guided(res, 0.3, 2.0)
    assert np.array_equal(g64[EDGE], c[EDGE].astype(np.float64)), what       # the formula returns c there
    assert_bits_equal(res[2][EDGE].float(), torch.from_numpy(c[EDGE]).to(res[2].dtype).float(), what + ": c")

    def one_nan(arr):
        """one NaN in one sample"""
        arr["ec"][EDGE, 8192 + 5] = np.nan
    for form, px0 in ((0, True), (1, False)):
        res, what = case(one_nan, px0=px0, form=form)
        g64, _ = fp64_guided(res, 0.3, 2.0)
        assert np.isnan(g64[EDGE]).all() and torch.isnan(res[2][EDGE].float()).all(), what
        if res[3] is not None:
            assert torch.isnan(res[3][EDGE].float()).all(), what

    if md != torch.float16:          # (fp16 outputs cannot reach a guidance difference beyond fp32)
        def overflow(arr):
            """out_c - out_u of +-3e38 (flow: R = inf); other parameterisations at the same values"""
            arr["xe"][EDGE, :64] = 0.0
            arr["ec"][EDGE, :64], arr["eu"][EDGE, :64] = -3e38, 3e38
            arr["ec"][EDGE, 64:128], arr["eu"][EDGE, 64:128] = 3e38, -3e38
        case(overflow)
        case(overflow, eta=0.0, r=0.0)

    def inf_r_bypassed(arr):
        """inf in R on a bypassed row (scale 1): the row's output is c"""
        arr["rp"][EDGE, :16] = np.inf
        arr["rp"][EDGE, 16:32] = -np.inf
        arr["rp"][EDGE, 32] = np.nan
    for form, px0 in ((0, True), (1, True), (1, False)):
        res, what = case(inf_r_bypassed, beta=-0.5, scales=[W, 1.0, -2.0], px0=px0, form=form)
        assert not torch.isfinite(res[1][EDGE]).all(), what
        if px0:
            _, c = fp64_guided(res, 0.3, 2.0, [W, 1.0, -2.0])
            assert_bits_equal(res[2][EDGE].float(), torch.from_numpy(c[EDGE]).to(res[2].dtype).float(), what + ": c")

    def tiny_threshold(arr):
        """the smallest positive threshold"""
    case(tiny_threshold, r=1e-45)
    case(tiny_threshold, r=1e-45, beta=0.3, eta=0.0)
