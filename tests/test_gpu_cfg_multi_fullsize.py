"""Multi-condition guidance (dpm_step_multi, dpm_replicate) at full size and beyond 2^31 elements, checked through
properties that do not depend on size (the numpy executor would take minutes there): the fused step equals the same
chain written as separate torch CUDA ops bit for bit, every replica equals out, and the threshold equals the quantile
taken on the materialised combined noise."""
import numpy as np
import pytest
import torch

from dpm_solver_b200._lib import FORM_DIFF2, FORM_LIN1, FORM_MS3, FORM_NONE
from dpm_solver_b200.ops import StepArgs
from test_gpu_fullsize import CO, eager_ms3

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SC = {2: (7.5, -2.0), 4: (3.0, 1.0, -0.5, 0.0)}
ALPHA, SIGMA = 0.83, 0.55


def _quantile_ref(xf, e, B, ps):
    """torch.quantile(|x0|, 0.995, dim=1).clamp_min(1) per sample (:422-423), as test_gpu_fullsize takes it: order
    statistics from torch.sort in groups of 256 samples, their interpolation from ATen's CPU lerp."""
    pos = np.float32(0.995) * np.float32(ps - 1)
    lo = int(np.floor(pos))
    w = float(np.float32(pos - np.float32(lo)))
    out = []
    for r in range(0, B, 256):
        x0 = ((xf[r:r + 256] - SIGMA * e[r:r + 256]) / torch.tensor([ALPHA], device=DEV)).reshape(-1, ps).abs()
        srt = torch.sort(x0, dim=1).values
        out.append(torch.maximum(torch.lerp(srt[:, lo].cpu(), srt[:, lo + 1].cpu(), torch.tensor(w)),
                                 torch.tensor(1.0)))
        del x0, srt
    return torch.cat(out)


def _fused_vs_eager(be, shape, dt, K, form, thr):
    g = torch.Generator(device=DEV).manual_seed(10 * K + form)
    mk = lambda s=1.0: (torch.randn(shape, device=DEV, generator=g) * s).to(dt)
    x, eu, m1 = mk(), mk(), mk()
    m2 = mk() if form == FORM_MS3 else None
    ecs = tuple(mk(1.0 + 0.2 * k) for k in range(K))
    B, ps = shape[0], x.numel() // shape[0]
    base = dict(n_model=2, e_uncond=eu, e_cond=ecs[0], e_conds=ecs, scales=SC[K], alpha_e=ALPHA, sigma_e=SIGMA,
                per_sample=ps)
    # the eager chain in fp32, one rounding per op; the division by a 1-element tensor is true division
    xf, euf = x.float(), eu.float()
    eps = euf
    for s, e in zip(SC[K], ecs):
        eps = eps + s * (e.float() - euf)
    q = None
    if thr:
        # the combined noise materialised in fp32 (FORM_NONE), and the per-sample threshold the quantile takes on it
        e, _ = be.step(StepArgs(form=FORM_NONE, state_dtype=torch.float32, want_m_out=True, **base))
        assert torch.equal(e, eps)
        q = be.dynamic_threshold(StepArgs(form=FORM_NONE, n_model=1, e_cond=e, xe=x, predict_x0=True, alpha_e=ALPHA,
                                          sigma_e=SIGMA, per_sample=ps, state_dtype=dt), 0.995, 1.0)
        assert torch.equal(q.cpu(), _quantile_ref(xf, e, B, ps))
        del e
    reps = tuple(torch.full_like(x, float("nan")) for _ in range(K))
    m, o = be.step(StepArgs(form=form, x=x, xe=x, m1=m1, m2=m2, predict_x0=True, want_m_out=True, state_dtype=dt,
                            thr=q, replicas=reps, **base, **CO))
    x0 = (xf - SIGMA * eps) / torch.tensor([ALPHA], device=DEV)
    del eps
    if thr:
        s = q.view(-1, *([1] * (x.dim() - 1)))
        x0 = x0.clamp(-s, s) / s
    assert torch.equal(m, x0.to(dt))
    T0 = x0.to(dt).float()
    del x0
    if form == FORM_MS3:
        ref = eager_ms3(xf, T0, m1.float(), m2.float(), CO)
    else:
        ref = (CO["a"] * xf + CO["c0"] * T0) + CO["c1"] * (CO["w0"] * (T0 - m1.float()))
    assert torch.equal(o, ref.to(dt))
    for r in reps:
        assert torch.equal(r, o)


@pytest.mark.parametrize("thr", [False, True])
@pytest.mark.parametrize("form", [FORM_MS3, FORM_DIFF2])
@pytest.mark.parametrize("K", [2, 4])
def test_multi_step_bf16_full_size_equals_eager_chain(cuda_backend, K, form, thr):
    """bench_multicond.py's shape: bf16 [2048, 4, 64, 64]."""
    _fused_vs_eager(cuda_backend, (2048, 4, 64, 64), torch.bfloat16, K, form, thr)


def test_multi_step_fp32_full_size_equals_eager_chain(cuda_backend):
    _fused_vs_eager(cuda_backend, (1024, 3, 256, 256), torch.float32, 2, FORM_MS3, True)


def test_multi_step_and_replicate_beyond_2_31_elements(cuda_backend):
    """More than 2^31 elements in one call (64-bit element offsets, 32-bit packet indices, a ragged tail): one LIN1
    multi-condition step written in place over x with both replicas, then a 3-way dpm_replicate of 2^31 + 8000
    elements (whole 16-byte words, the vector kernel), checked on slices at the start, across element 2^31 and at the
    tail. Both conditions share one storage with different scales. At most five 4.3 GB bf16 tensors are alive at a time
    (peak <= 25 GiB)."""
    n = (1 << 31) + 8 * 1000 + 3
    torch.cuda.reset_peak_memory_stats()
    g = torch.Generator(device=DEV).manual_seed(4)
    x = torch.randn(n, device=DEV, generator=g, dtype=torch.bfloat16)
    eu = torch.randn(n, device=DEV, generator=g, dtype=torch.bfloat16)
    ec = torch.randn(n, device=DEV, generator=g, dtype=torch.bfloat16)
    spots = [slice(0, 4096), slice((1 << 31) - 2048, (1 << 31) + 2048), slice(n - 3000, n)]
    s1, s2, A, c0 = 7.5, -2.0, 0.9375, -0.40625
    want = []
    for sl in spots:
        euf, ecf = eu[sl].float(), ec[sl].float()
        T0 = ((euf + s1 * (ecf - euf)) + s2 * (ecf - euf)).bfloat16().float()
        want.append((A * x[sl].float() + c0 * T0).bfloat16())
    reps = (torch.empty_like(x), torch.empty_like(x))
    m, o = cuda_backend.step(StepArgs(form=FORM_LIN1, n_model=2, x=x, e_uncond=eu, e_cond=ec, e_conds=(ec, ec),
                                      scales=(s1, s2), a=A, c0=c0, state_dtype=torch.bfloat16, out=x, replicas=reps))
    assert m is None and o is x
    for sl, w in zip(spots, want):
        assert torch.equal(x[sl], w), sl
        for r in reps:
            assert torch.equal(r[sl], w), sl
    del reps, eu, ec, m, o
    nv = n - 3                        # whole 16-byte words: the vector kernel, not the copy fallback
    xx = x[:nv].view(1, nv)
    cp = cuda_backend.replicate(xx, 3)
    assert cp.shape == (3, nv)
    for sl in spots[:2] + [slice(nv - 3000, nv)]:
        for c in range(3):
            assert torch.equal(cp[c, sl], x[sl]), (c, sl)
    del cp, xx, x
    assert torch.cuda.max_memory_allocated() <= 25 * 2 ** 30
