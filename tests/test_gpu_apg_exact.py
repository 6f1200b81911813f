"""Adaptive projected guidance on the H100, bit for bit: the words of dpm_apg_words against the exact mirror of words.cu
(apg_oracle.apg_words_exact) on every dtype pair, on sample sizes that end inside a packet, at a chunk edge and past it,
on the vector and the element-wise path, with and without momentum (R too), with per-sample scales and channels_last;
the merge order of a sample's chunks; the coefficient block (dev_coef) of the adaptive controller feeding both the words
pass and k_step_scalar_apg while the host values are the (1, 0) that the solver passes; the per-sample threshold of both
step kernels."""
import dataclasses

import numpy as np
import pytest
import torch

from apg_oracle import APGOracle, apg_final, apg_sums_exact
from step_edges import assert_bits_equal
from test_gpu_apg import COEF, DT, PAIRS, _args, cpu

pytestmark = pytest.mark.gpu
PER_SAMPLE = [7, 9, 104, 8192, 8193, 8192 * 3 - 8, 16384, 3 * 8192 + 1]
SETTINGS = [(0.0, 0.0), (0.3, 1.0), (1.0, 1e6), (0.5, 40.0)]      # (eta, norm_threshold): off, clips, never clips, some


def unaligned(t):
    """The same values one element into a larger buffer: a view the vector paths cannot take."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    return v


def like_launch(a, gen):
    """An fp32 tensor of random values laid out like the launch (xe)."""
    r = torch.randn(a.xe.shape, generator=gen).cuda()
    return r.contiguous(memory_format=torch.channels_last) if not a.xe.is_contiguous() else r


def check_words(be, a, eta, r, beta, gen, what):
    r_prev = like_launch(a, gen) if beta else None
    r_out = torch.empty_like(r_prev) if beta else None
    w = be.apg_words(a, eta, r, beta, r_prev, r_out)
    ro = torch.empty(a.xe.shape) if beta else None
    want = APGOracle(exact=True).apg_words(cpu(a), eta, r, beta, None if r_prev is None else r_prev.cpu(), ro)
    assert_bits_equal(w, want, what + ": words")
    if beta:
        assert_bits_equal(r_out, ro, what + ": R")
    return w, r_out


@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", PER_SAMPLE)
def test_words_bit_exact(cuda_backend, pair, ps):
    gen = torch.Generator().manual_seed(ps)
    k = 0
    for path in ("vector", "element-wise"):
        for beta in (0.0, -0.5):
            for per_sample in (False, True):
                param = k % 6
                eta, r = SETTINGS[k % len(SETTINGS)]
                k += 1
                a = _args(param, True, DT[pair[0]], DT[pair[1]], 3, ps, gen, per_sample=per_sample)
                if path == "element-wise":
                    a.e_uncond = unaligned(a.e_uncond)
                check_words(cuda_backend, a, eta, r, beta, gen, "%s param %d beta %g per_sample %s" % (
                    path, param, beta, per_sample))


@pytest.mark.parametrize("ps", [8192, 16384])
def test_words_bit_exact_channels_last(cuda_backend, ps):
    """A channels_last launch sums each sample in its storage order, (h, w, c)."""
    gen = torch.Generator().manual_seed(ps + 1)
    for pair in PAIRS:
        for beta in (0.0, 0.3):
            a = _args(4 if beta else 0, True, DT[pair[0]], DT[pair[1]], 2, ps, gen, layout="cl", per_sample=True)
            assert not a.xe.is_contiguous()
            check_words(cuda_backend, a, 0.3, 40.0, beta, gen, "%s-%s beta %g" % (pair + (beta,)))


def test_chunks_merge_in_chunk_order(cuda_backend):
    """<R, c> of chunk 0 is +2^63 and that of chunk 1 exactly -2^63; chunk 2 holds ordinary values. Merged in chunk
    order, chunk 2's part survives; merged in another order it is absorbed by 2^63. So the merge order, invisible in
    the words on ordinary data (an fp64 sum reordered moves them by far less than an fp32 ulp), shows in their bits."""
    from dpm_solver_b200.ops import StepArgs
    ps, Bn = 3 * 8192, 2
    gen = torch.Generator().manual_seed(11)
    xe, ec, eu = torch.zeros(Bn, ps), torch.zeros(Bn, ps), torch.zeros(Bn, ps)
    # flow with sigma = 1: c = xe - out. xe = 0, out_c = -1: c = 1; out_u = +-2^50: R = 1 +- 2^50 = +-2^50 exactly
    ec[:, :16384] = -1.0
    eu[:, :8192], eu[:, 8192:16384] = 2.0 ** 50, -2.0 ** 50
    for t in (xe, ec, eu):
        t[:, 16384:] = torch.randn(Bn, 8192, generator=gen)
    a = StepArgs(form=0, n_model=2, xe=xe.cuda(), e_cond=ec.cuda(), e_uncond=eu.cuda(), param=4, predict_x0=True,
                 guidance=4.0, alpha_e=1.0, sigma_e=1.0, alpha_t=1.0, sigma_t=1.0, state_dtype=torch.float32,
                 per_sample=ps)
    o = APGOracle(exact=True)
    c = o._x0(cpu(a), ec.numpy(), xe.numpy())
    R = (c - o._x0(cpu(a), eu.numpy(), xe.numpy())).astype(np.float32)
    assert (R[:, :8192] == 2.0 ** 50).all() and (R[:, 8192:16384] == -2.0 ** 50).all()
    per_chunk = [apg_sums_exact(R[:, k * 8192:(k + 1) * 8192], c[:, k * 8192:(k + 1) * 8192]) for k in range(3)]

    def merged(order):
        tot = [np.zeros(Bn) for _ in range(3)]
        for k in order:
            tot = [t + s for t, s in zip(tot, per_chunk[k])]
        return apg_final(*tot, np.full(Bn, 4.0), 0.0, 0.0)
    want = o.apg_words(cpu(a), 0.0, 0.0, 0.0)
    assert np.array_equal(merged([0, 1, 2]), want.numpy())
    for order in ([2, 1, 0], [0, 2, 1], [2, 0, 1]):
        assert not np.array_equal(merged(order)[0], want.numpy()[0]), order   # the data tells the orders apart
    assert_bits_equal(cuda_backend.apg_words(a, 0.0, 0.0, 0.0), want, "words")


# ---- the coefficient block of the device controller ----------------------------------------------------------------

def block_marginals(param):
    """(alpha, sigma) of a real schedule at t = 0.37, as the adaptive controller writes them to dev_coef[9..10]."""
    from test_apg import product_schedule
    ns = product_schedule("flow" if param == 4 else "noise")
    t = torch.tensor([0.37])
    return float(ns.marginal_alpha(t)), float(ns.marginal_std(t))


@pytest.mark.parametrize("pair", [("f32", "f32"), ("bf16", "bf16"), ("f16", "f32")], ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("param", range(6))
def test_dev_coef_words_and_scalar_step(cuda_backend, pair, param):
    """The words pass and k_step_scalar_apg take alpha, sigma from the block, not from the host's (1, 0); an EDM
    launch, whose words are not marginals, is refused with a block and launches nothing."""
    gen = torch.Generator().manual_seed(20 + param)
    al, sg = block_marginals(param)
    n = 0
    for form in (0, 1, 5):
        for px0 in (True, False):
            for beta, per_sample in ((0.0, False), (-0.5, True)):
                a = _args(param, px0, DT[pair[0]], DT[pair[1]], 3, 3 * 40, gen, form, per_sample=per_sample)
                v = [COEF[k] for k in ("a", "c0", "c1", "c2", "w0", "w1", "w2", "w3", "w4")] + [al, sg]
                a.coef_dev = torch.tensor(v + [0.] * 5, dtype=torch.float32).cuda()
                a.alpha_e, a.sigma_e, a.alpha_t, a.sigma_t = 1.0, 0.0, 1.0, 0.0     # what _apg_args passes
                if param == 5:
                    from dpm_solver_b200._lib import DpmLibraryError
                    before = cuda_backend.launch_count()
                    with pytest.raises(DpmLibraryError, match="dev_coef"):
                        cuda_backend.apg_words(a, 0.3, 2.0, 0.0)
                    a.apg_words = torch.ones(2, 3).cuda()
                    with pytest.raises(DpmLibraryError, match="dev_coef"):
                        cuda_backend.step(a)
                    assert cuda_backend.launch_count() == before
                    return
                r_prev = like_launch(a, gen) if beta else None
                r_out = torch.empty_like(r_prev) if beta else None
                words = cuda_backend.apg_words(a, 0.3, 2.0, beta, r_prev, r_out)
                c = dataclasses.replace(cpu(a), alpha_e=al, sigma_e=sg, alpha_t=al, sigma_t=sg)
                ro = torch.empty(a.xe.shape) if beta else None
                want = APGOracle(exact=True).apg_words(c, 0.3, 2.0, beta, None if r_prev is None else r_prev.cpu(), ro)
                what = "form %d predict_x0 %s beta %g" % (form, px0, beta)
                assert_bits_equal(words, want, what + ": words")
                if beta:
                    assert_bits_equal(r_out, ro, what + ": R")
                a.apg_words, a.apg_r = words, r_out
                c.apg_words, c.apg_r = want, ro
                m, o = cuda_backend.step(a)
                mw, ow = APGOracle(exact=True).step(c)
                assert_bits_equal(m, mw, what + ": model value")
                if ow is not None:
                    assert_bits_equal(o, ow, what + ": update")
                n += 1
    assert n == 12


# ---- the per-sample threshold --------------------------------------------------------------------------------------

@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: "%s-%s" % p)
@pytest.mark.parametrize("ps", [16 * 64, 3 * 37])     # k_step_direct_apg / k_step_scalar_apg
def test_thresholded_step_reads_its_sample_threshold(cuda_backend, pair, ps):
    gen = torch.Generator().manual_seed(ps + 3)
    Bn = 5
    for form in (0, 1, 3):
        for param in range(6):
            a = _args(param, True, DT[pair[0]], DT[pair[1]], Bn, ps, gen, form, per_sample=form == 3)
            a.thr = torch.tensor([1.5, 0.7, 2.5, 1.1, 0.9], dtype=torch.float32).cuda()
            a.apg_words = cuda_backend.apg_words(a, 0.2, 3.0, 0.0)
            m, o = cuda_backend.step(a)
            mw, ow = APGOracle(exact=True).step(cpu(a))
            assert_bits_equal(m, mw, "form %d param %d: model value" % (form, param))
            if ow is not None:
                assert_bits_equal(o, ow, "form %d param %d: update" % (form, param))
