"""GPU parity tests: every kernel form of libdpmsolver_b200.so against the numpy executor, bit for bit
(fp32 storage: identical to the reference's unfused fp32 op chain; bf16/f16 storage: fp32 math,
one round-to-nearest-even on store). All calls go through the C-ABI."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from dpm_solver_b200 import _lib, ops
from dpm_solver_b200._lib import (FORM_DIFF2, FORM_LIN1, FORM_LIN2, FORM_LIN3, FORM_MS3, FORM_NONE, FORM_SS3T,
                                  PARAM_NOISE, PARAM_SCORE, PARAM_V, PARAM_X_START)
from dpm_solver_b200.ops import StepArgs
from oracle_backend import OracleBackend

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FORMS = [FORM_LIN1, FORM_LIN2, FORM_LIN3, FORM_DIFF2, FORM_MS3, FORM_SS3T]


def rnd(n, seed, dtype=torch.float32, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * scale).to(dtype)


def coeffs(form, seed=0):
    r = np.random.RandomState(seed)
    v = r.uniform(0.2, 1.5, size=9).astype(np.float32) * r.choice([-1, 1], size=9)
    return dict(a=float(v[0]), c0=float(v[1]), c1=float(v[2]), c2=float(v[3]), w0=float(v[4]), w1=float(v[5]),
                w2=float(abs(v[6])), w3=float(abs(v[7])), w4=float(abs(v[8]) + 0.1))


def make_args(form, n_model, n, sdt, mdt, param=PARAM_NOISE, predict_x0=False, sep_xe=False, thr=None,
              per_sample=0, c0_on_old=False, want_m=True, seed=0):
    kw = coeffs(form, seed)
    a = StepArgs(form=form, n_model=n_model, param=param, predict_x0=predict_x0, c0_on_old=c0_on_old,
                 guidance=7.5, alpha_e=0.83, sigma_e=0.55, want_m_out=want_m, state_dtype=sdt, **kw)
    if form != FORM_NONE:
        a.x = rnd(n, seed + 1, sdt)
    if n_model == 0:
        a.m0 = rnd(n, seed + 2, sdt)
    else:
        a.e_cond = rnd(n, seed + 3, mdt)
        if n_model == 2:
            a.e_uncond = rnd(n, seed + 4, mdt)
        if predict_x0 or param in (PARAM_X_START, PARAM_V):
            a.xe = rnd(n, seed + 5, sdt) if (sep_xe or form == FORM_NONE) else a.x
    if form in (FORM_LIN2, FORM_LIN3, FORM_DIFF2, FORM_MS3, FORM_SS3T):
        a.m1 = rnd(n, seed + 6, sdt)
    if form in (FORM_LIN3, FORM_MS3, FORM_SS3T):
        a.m2 = rnd(n, seed + 7, sdt)
    if thr is not None:
        a.thr, a.per_sample = thr, per_sample
    return a


def to_dev(a):
    import copy
    b = copy.copy(a)
    for f in ("x", "xe", "m0", "m1", "m2", "e_cond", "e_uncond", "thr"):
        v = getattr(a, f)
        if v is not None:
            setattr(b, f, v.to(DEV))
    if a.xe is not None and a.xe is a.x:
        b.xe = b.x
    return b


def check(a, cuda_backend):
    ref_m, ref_o = OracleBackend().step(a)
    got_m, got_o = cuda_backend.step(to_dev(a))
    torch.cuda.synchronize()
    for r, g, what in ((ref_m, got_m, "m_out"), (ref_o, got_o, "out")):
        assert (r is None) == (g is None), what
        if r is not None:
            assert g.dtype == r.dtype
            assert torch.equal(g.cpu().view(torch.int16 if r.element_size() == 2 else torch.int32),
                               r.view(torch.int16 if r.element_size() == 2 else torch.int32)), what


@pytest.mark.parametrize("sdt", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("form", FORMS)
def test_pure_updates_bit_exact(cuda_backend, form, sdt):
    for n in (8 * 4096 + 5, 7, 8 * 148 * 512 * 2 + 8):      # tail, tiny, > one persistent wave
        check(make_args(form, 0, n, sdt, sdt, c0_on_old=(n == 7), seed=form), cuda_backend)


@pytest.mark.parametrize("sdt,mdt", [(torch.float32, torch.float32), (torch.bfloat16, torch.bfloat16),
                                     (torch.float16, torch.float16), (torch.float32, torch.bfloat16),
                                     (torch.float32, torch.float16), (torch.bfloat16, torch.float32)])
@pytest.mark.parametrize("form", [FORM_NONE, FORM_LIN1, FORM_DIFF2, FORM_MS3, FORM_SS3T, FORM_LIN3])
def test_post_model_steps_bit_exact(cuda_backend, form, sdt, mdt):
    n = 8 * 3000 + 3
    for n_model, param, px0, sep in itertools.product((1, 2), (PARAM_NOISE, PARAM_X_START, PARAM_V, PARAM_SCORE),
                                                      (False, True), (False, True)):
        if sep and form == FORM_NONE:
            continue
        check(make_args(form, n_model, n, sdt, mdt, param=param, predict_x0=px0, sep_xe=sep,
                        c0_on_old=bool(n_model == 2), seed=form * 7 + n_model), cuda_backend)


def test_thresholding_clamp_bit_exact(cuda_backend):
    for per_sample, B in ((3 * 16 * 16, 6), (1001, 5)):     # packet-aligned and ragged samples
        n = per_sample * B
        thr = torch.tensor(np.linspace(0.4, 2.5, B), dtype=torch.float32)
        for form in (FORM_NONE, FORM_MS3):
            for sdt in (torch.float32, torch.bfloat16):
                check(make_args(form, 2, n, sdt, sdt, predict_x0=True, thr=thr, per_sample=per_sample, seed=11),
                      cuda_backend)


def test_misaligned_and_noncontiguous(cuda_backend):
    """Odd element offsets take the generic kernel; results are identical."""
    n = 8 * 1000
    a = make_args(FORM_MS3, 0, n + 1, torch.float32, torch.float32, seed=3)
    ref = OracleBackend().step(StepArgs(**{**a.__dict__, "x": a.x[1:], "m0": a.m0[1:], "m1": a.m1[1:], "m2": a.m2[1:]}))[1]
    d = to_dev(a)
    got = cuda_backend.step(StepArgs(**{**d.__dict__, "x": d.x[1:], "m0": d.m0[1:], "m1": d.m1[1:], "m2": d.m2[1:]}))[1]
    assert torch.equal(got.cpu(), ref)
    xs = torch.randn(64, 33, device=DEV)[:, :32]             # non-contiguous view
    m = torch.randn(64, 32, device=DEV)
    got = ops.lincomb(xs, [m], 0.5, [2.0])
    assert torch.equal(got, 0.5 * xs + 2.0 * m)


def test_in_place_alias(cuda_backend):
    x = torch.randn(8 * 5000, device=DEV)
    m = torch.randn(8 * 5000, device=DEV)
    ref = 0.7 * x + (-0.2) * m
    ops.lincomb(x, [m], 0.7, [-0.2], out=x)
    assert torch.equal(x, ref)


@pytest.mark.parametrize("sdt,mdt", [(torch.float32, torch.float32), (torch.bfloat16, torch.bfloat16), (torch.float32, torch.bfloat16),
                                     (torch.float16, torch.float16)])
def test_tma_variant_equals_direct(cuda_backend, sdt, mdt):
    """variant 1 (cp.async.bulk shared-memory ring) must be bitwise identical to variant 0."""
    n = 8 * (148 * 512 * 3 + 77) + 4
    cases = [make_args(f, 0, n, sdt, sdt, seed=f) for f in FORMS]
    cases += [make_args(f, nm, n, sdt, mdt, predict_x0=True, seed=f + nm) for f in (FORM_NONE, FORM_LIN1, FORM_DIFF2, FORM_MS3) for nm in (1, 2)]
    cases += [make_args(f, 2, n, sdt, mdt, predict_x0=True, sep_xe=True, param=PARAM_V, seed=f) for f in (FORM_DIFF2, FORM_SS3T, FORM_LIN3)]
    thr = torch.tensor(np.linspace(0.5, 2.0, 4), dtype=torch.float32)
    cases.append(make_args(FORM_MS3, 1, 8 * 4096, sdt, mdt, predict_x0=True, thr=thr, per_sample=8 * 1024, seed=5))
    for a in cases:
        d = to_dev(a)
        cuda_backend.set_tuning(0, 0, 0)
        m0, o0 = cuda_backend.step(d)
        for threads, ctas in ((256, 1), (128, 2), (512, 1), (0, 0)):
            cuda_backend.set_tuning(1, threads, ctas)
            m1, o1 = cuda_backend.step(d)
            torch.cuda.synchronize()
            for p, q in ((m0, m1), (o0, o1)):
                assert (p is None) == (q is None)
                if p is not None:
                    assert torch.equal(p, q)
    cuda_backend.set_tuning(2, 0, 0)


@pytest.mark.parametrize("threads,ctas", [(128, 4), (256, 8), (512, 2), (64, 16)])
def test_direct_tuning_is_result_invariant(cuda_backend, threads, ctas):
    a = to_dev(make_args(FORM_MS3, 2, 8 * 100003, torch.bfloat16, torch.bfloat16, predict_x0=True, seed=9))
    cuda_backend.set_tuning(0, 0, 0)
    m0, o0 = cuda_backend.step(a)
    cuda_backend.set_tuning(0, threads, ctas)
    m1, o1 = cuda_backend.step(a)
    cuda_backend.set_tuning(2, 0, 0)
    assert torch.equal(m0, m1) and torch.equal(o0, o1)


# ---- quantile ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_sample,B", [(24, 300), (1000, 9), (4 * 64 * 64, 37), (3 * 256 * 256, 5), (3 * 512 * 512, 2), (1 << 21, 2)])
@pytest.mark.parametrize("sdt,mdt,nm", [(torch.float32, torch.float32, 1), (torch.float32, torch.float32, 2),
                                        (torch.bfloat16, torch.bfloat16, 2), (torch.float32, torch.bfloat16, 1)])
def test_dynamic_threshold_exact(cuda_backend, per_sample, B, sdt, mdt, nm):
    from oracle import dpm_oracle as O
    n = per_sample * B
    a = make_args(FORM_NONE, nm, n, sdt, mdt, predict_x0=True, seed=per_sample % 97)
    a.per_sample = per_sample
    import os
    x0 = OracleBackend()._model_value(a, None).reshape(B, -1)
    for q, max_val in ((0.995, 1.0), (0.5, 0.1), (1.0, 0.0), (0.0, 0.0), (0.97, 0.0)):
        ref = np.maximum(O.quantile_abs(x0, q), np.float32(max_val))
        for impl in ("pipeline", "cluster"):     # streaming pipeline (default) and the cluster radix kernel
            os.environ["DPM_QUANTILE_IMPL"] = impl
            try:
                got = cuda_backend.dynamic_threshold(to_dev(a), q, max_val).cpu().numpy()
            finally:
                os.environ.pop("DPM_QUANTILE_IMPL", None)
            np.testing.assert_array_equal(got, ref, err_msg=f"{impl} q={q}")


def test_dynamic_threshold_ties_and_constants(cuda_backend):
    """Heavy ties (quantised values, all-equal samples, zeros) select the same order statistics."""
    from oracle import dpm_oracle as O
    for per_sample, B in ((4096, 6), (16384, 6), (3 * 128 * 128, 5)):   # exact path / bracket path (1 CTA, cluster)
        x = (torch.randn(B, per_sample, generator=torch.Generator().manual_seed(1)) * 4).round() / 4
        x[1] = 0.75
        x[2] = 0.0
        x[3, : per_sample // 2] = 9.5      # half the sample tied at the top
        a = StepArgs(form=FORM_NONE, n_model=1, e_cond=torch.zeros(B * per_sample), xe=x.reshape(-1), predict_x0=True,
                     alpha_e=1.0, sigma_e=0.0, per_sample=per_sample, state_dtype=torch.float32)
        for q in (0.995, 0.25, 0.9999, 0.75):
            got = cuda_backend.dynamic_threshold(to_dev(a), q, 0.0).cpu().numpy()
            np.testing.assert_array_equal(got, O.quantile_abs(x.numpy(), q))


def _plain_x0(x):
    """StepArgs whose x0 is x itself: noise network, eps = 0, alpha 1, sigma 0."""
    B, ps = x.shape
    return StepArgs(form=FORM_NONE, n_model=1, e_cond=torch.zeros(B * ps), xe=x.reshape(-1).contiguous(), predict_x0=True,
                    alpha_e=1.0, sigma_e=0.0, per_sample=ps, state_dtype=torch.float32)


def test_dynamic_threshold_pivot_defeating_sample(cuda_backend):
    """k_q_pivots reads 256 groups of 4 consecutive elements at a stride of per_sample/256 = 64: a sample whose
    elements 64k..64k+3 are small and all others large hides the target rank from the pivots. The exact counts then
    refuse the bracket and the finish kernel selects over the whole sample (path 2); the result is still exact."""
    from oracle import dpm_oracle as O
    ps, B = 16384, 3
    g = torch.Generator().manual_seed(8)
    x = 10.0 + torch.rand(B, ps, generator=g) * 5.0
    probe = (torch.arange(ps) % 64) < 4
    x[:, probe] = torch.rand(B, int(probe.sum()), generator=g)
    for q in (0.995, 0.5):
        got, hdr = cuda_backend.dynamic_threshold(to_dev(_plain_x0(x)), q, 0.0, return_stats=True)
        assert (hdr[:, 4] == 2).all(), hdr[:, 4]
        np.testing.assert_array_equal(got.cpu().numpy(), O.quantile_abs(x.numpy(), q))


def test_dynamic_threshold_count_cta_overflow(cuda_backend):
    """One count CTA (16384 elements at the default shape) meets more bracket keys than its block-local list holds
    (kLocalCand = 2048) while the sample's bracket count stays within the candidate capacity (16384/16 + 2048 = 3072):
    2500 ties span the 0.995 rank. The CTA poisons the count (bit 30 of header word 3), which forces the exact fallback
    (path 2) rather than a select over an incomplete candidate list."""
    from oracle import dpm_oracle as O
    ps, B, ties, below = 16384, 2, 2500, 13850
    g = torch.Generator().manual_seed(9)
    x = torch.empty(B, ps)
    for b in range(B):
        v = torch.cat([torch.rand(below, generator=g), torch.full((ties,), 5.0),
                       6.0 + torch.rand(ps - below - ties, generator=g)])
        x[b] = v[torch.randperm(ps, generator=g)] * torch.where(torch.rand(ps, generator=g) < 0.5, -1.0, 1.0)
    lo = int(np.floor(np.float32(0.995) * np.float32(ps - 1)))
    assert below <= lo and lo + 1 < below + ties                   # both order statistics are tied keys
    got, hdr = cuda_backend.dynamic_threshold(to_dev(_plain_x0(x)), 0.995, 0.0, return_stats=True)
    words = hdr[:, 3].cpu().numpy().view(np.uint32)
    assert ((words & (1 << 30)) != 0).all(), words
    assert ((words & ((1 << 30) - 1)) <= 3072).all(), words      # within capacity: only the poison forces the fallback
    assert (hdr[:, 4] == 2).all(), hdr[:, 4]
    np.testing.assert_array_equal(got.cpu().numpy(), O.quantile_abs(x.numpy(), 0.995))


def test_quantile_golden(golden, cuda_backend):
    """Directly against torch.quantile outputs recorded from the reference's code path."""
    g = golden["glue"]
    tiny = torch.from_numpy(g["tiny"]) * 3.0
    a = StepArgs(form=FORM_NONE, n_model=1, e_cond=torch.zeros(tiny.numel()), xe=tiny.reshape(-1).contiguous(),
                 predict_x0=True, alpha_e=1.0, sigma_e=0.0, per_sample=tiny.shape[1], state_dtype=torch.float32)
    got = cuda_backend.dynamic_threshold(to_dev(a), 0.995, 0.0).cpu().numpy()
    np.testing.assert_array_equal(got, g["tiny_q"])
    from cases import seeded
    big = seeded((3, 3 * 64 * 64), 203)
    a = StepArgs(form=FORM_NONE, n_model=1, e_cond=torch.zeros(big.numel()), xe=big.reshape(-1).contiguous(),
                 predict_x0=True, alpha_e=1.0, sigma_e=0.0, per_sample=big.shape[1], state_dtype=torch.float32)
    got = cuda_backend.dynamic_threshold(to_dev(a), 0.995, 0.0).cpu().numpy()
    np.testing.assert_array_equal(got, g["big_q"])


# ---- named C-ABI entry points --------------------------------------------------------------------------
def test_named_entry_points(cuda_backend):
    L = _lib.lib()
    n = 8 * 2048 + 6
    x, m0, m1, m2 = (rnd(n, 40 + i).to(DEV) for i in range(4))
    out = torch.empty_like(x)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    ob = OracleBackend()
    cpu = lambda t: t.cpu()

    _lib.check(L.dpm_solver_first_update(p(out), p(x), p(m0), 0.9, -0.3, n, 0, st))
    ref = ob.step(StepArgs(form=FORM_LIN1, x=cpu(x), m0=cpu(m0), a=0.9, c0=-0.3))[1]
    assert torch.equal(out.cpu(), ref)

    _lib.check(L.dpm_multistep_second_update(p(out), p(x), p(m0), p(m1), 0.9, -0.3, 0.15, 1.1, n, 0, st))
    ref = ob.step(StepArgs(form=FORM_DIFF2, x=cpu(x), m0=cpu(m0), m1=cpu(m1), a=0.9, c0=-0.3, c1=0.15, w0=1.1))[1]
    assert torch.equal(out.cpu(), ref)

    _lib.check(L.dpm_multistep_third_update(p(out), p(x), p(m0), p(m1), p(m2), 0.9, -0.3, 0.15, -0.02, 1.1, 0.9, 0.45, 0.5, n, 0, st))
    ref = ob.step(StepArgs(form=FORM_MS3, x=cpu(x), m0=cpu(m0), m1=cpu(m1), m2=cpu(m2), a=0.9, c0=-0.3, c1=0.15,
                           c2=-0.02, w0=1.1, w1=0.9, w2=0.45, w3=0.5))[1]
    assert torch.equal(out.cpu(), ref)

    _lib.check(L.dpm_singlestep_diff_update(p(out), p(x), p(m0), p(m1), 0.9, -0.3, 0.15, n, 0, st))
    ref = ob.step(StepArgs(form=FORM_DIFF2, x=cpu(x), m0=cpu(m1), m1=cpu(m0), a=0.9, c0=-0.3, c1=0.15, w0=1.0, c0_on_old=True))[1]
    assert torch.equal(out.cpu(), ref)

    _lib.check(L.dpm_singlestep_third_taylor_update(p(out), p(x), p(m0), p(m1), p(m2), 0.9, -0.3, 0.15, -0.02,
                                                    3.0, 1.5, 2 / 3, 1 / 3, 1 / 3, n, 0, st))
    ref = ob.step(StepArgs(form=FORM_SS3T, x=cpu(x), m0=cpu(m2), m1=cpu(m1), m2=cpu(m0), a=0.9, c0=-0.3, c1=0.15,
                           c2=-0.02, w0=3.0, w1=1.5, w2=2 / 3, w3=1 / 3, w4=1 / 3))[1]
    assert torch.equal(out.cpu(), ref)

    _lib.check(L.dpm_lincomb(p(out), p(x), p(m0), p(m1), p(m2), 3, 0.5, 0.25, -2.0, 1.5, n, 0, st))
    assert torch.equal(out, ((0.5 * x + 0.25 * m0) + (-2.0) * m1) + 1.5 * m2)

    _lib.check(L.dpm_cfg_combine(p(out), p(m0), p(m1), 7.5, n, 0, st))
    assert torch.equal(out, m0 + 7.5 * (m1 - m0))

    _lib.check(L.dpm_data_prediction(p(out), p(x), p(m0), 0.8, 0.6, None, 0, n, 0, st))
    xn, mn = x.cpu().numpy(), m0.cpu().numpy()
    np.testing.assert_array_equal(out.cpu().numpy(), (xn - np.float32(0.6) * mn) / np.float32(0.8))


def test_error_reporting(cuda_backend):
    L = _lib.lib()
    assert L.dpm_step(None, None) == -1
    assert b"NULL" in L.dpm_last_error()
    d = _lib.StepDesc()
    d.n, d.form, d.state_dtype = 64, FORM_MS3, 0
    assert L.dpm_step(C.byref(d), None) == -1                   # required tensors missing
    d.form = 99
    assert L.dpm_step(C.byref(d), None) == -1
    assert L.dpm_lincomb(None, None, None, None, None, 4, 1., 1., 1., 1., 8, 0, None) == -1
    assert L.dpm_set_tuning(3, 0, 0) == -1 and L.dpm_set_tuning(0, 100, 0) == -1
    assert L.dpm_set_tuning(2, 0, 0) == 0
    with pytest.raises(RuntimeError, match="CUDA-only"):
        ops.lincomb(torch.randn(8), [torch.randn(8)], 1.0, [1.0])
    with pytest.raises(TypeError):
        ops.lincomb(torch.randn(8, device=DEV).double(), [torch.randn(8, device=DEV).double()], 1.0, [1.0])
    with pytest.raises(ValueError):
        ops.lincomb(torch.randn(8, device=DEV), [torch.randn(9, device=DEV)], 1.0, [1.0])


def test_launch_counter(cuda_backend):
    before = cuda_backend.launch_count()
    x = torch.randn(8 * 100 + 3, device=DEV)
    ops.lincomb(x, [x], 1.0, [1.0])
    assert cuda_backend.launch_count() - before == 2            # packet body + scalar tail


def test_cuda_graph_capture(cuda_backend):
    """Scalars travel by value: a captured step replays with no host involvement."""
    n = 8 * 20000
    x, m0, m1, m2 = (torch.randn(n, device=DEV) for _ in range(4))
    out = torch.empty_like(x)
    a = StepArgs(form=FORM_MS3, x=x, m0=m0, m1=m1, m2=m2, out=out, **coeffs(FORM_MS3, 1))
    cuda_backend.step(a)
    ref = out.clone()
    out.zero_()
    gph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(gph, stream=s):
            cuda_backend.step(a)
    torch.cuda.current_stream().wait_stream(s)
    out.zero_()
    gph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ref)


def test_constant_division_is_ieee(cuda_backend):
    """The reciprocal-refinement division by a launch constant (common.cuh: div_const) must equal
    IEEE division bit for bit: ~1e9 (x, d) pairs -- random magnitudes over 60 binades, values
    next to powers of two, exact multiples, zeros / denormals / huge values (guarded IEEE path)."""
    n = 1 << 22
    g = torch.Generator(device=DEV).manual_seed(7)
    mant = torch.rand(n, device=DEV, generator=g) + 1.0
    expo = torch.randint(-30, 30, (n,), device=DEV, generator=g).float()
    sign = torch.randint(0, 2, (n,), device=DEV, generator=g).float() * 2 - 1
    x = (sign * mant * torch.exp2(expo)).contiguous()
    special = torch.tensor([0.0, -0.0, 1e-38, -1e-39, 1e-45, 3e38, -3e38, 1.0, 2.0, 0.5, 1.0000001, 0.99999994,
                            1e-26, -3e-25, 9.9e-26, 1.1e-25, 9e29, 1.1e30, float("inf"), -float("inf")], device=DEV)
    x[:special.numel()] = special
    zeros = torch.zeros_like(x)
    rs = np.random.RandomState(3)
    divisors = np.concatenate([rs.uniform(1e-3, 1.0, 150), rs.uniform(1.0, 40.0, 40), [1e-7, 3e-6, 2e6, 1e-30, 1e20],
                               [1.0, 0.5, 0.25, 2.0, 0.99999994, 1.0000001, 0.0029151, 0.9998, 0.33333334,
                                np.float32(1) - np.float32(2 ** -24), 1.9999999]]).astype(np.float32)
    xe = x.cpu().numpy()
    bad = 0
    for d in divisors:
        a = StepArgs(form=FORM_NONE, n_model=1, e_cond=zeros, xe=x, predict_x0=True, alpha_e=float(d), sigma_e=0.0,
                     state_dtype=torch.float32)
        got = cuda_backend.step(a)[0].cpu().numpy()
        with np.errstate(all="ignore"):
            ref = (xe - np.float32(0.0) * np.float32(0.0)) / d
        bad += int((got.view(np.uint32) != ref.view(np.uint32)).sum())
        # multiples of d divide exactly
        xm = (x * float(d)).contiguous()
        a.xe = xm
        got = cuda_backend.step(a)[0].cpu().numpy()
        with np.errstate(all="ignore"):
            ref = xm.cpu().numpy() / d
        bad += int((got.view(np.uint32) != ref.view(np.uint32)).sum())
    assert bad == 0


@pytest.mark.parametrize("sdt", [torch.float32, torch.bfloat16])
def test_second_output_copy(cuda_backend, sdt):
    """out2 (the other half of the doubled CFG batch, model_wrapper :326) receives the same x_t."""
    for n in (8 * 200000 + 3, 8 * 700):
        for variant in (0, 1):
            a = make_args(FORM_DIFF2, 2, n, sdt, sdt, predict_x0=True, seed=21)
            ref_m, ref_o = OracleBackend().step(a)
            d = to_dev(a)
            buf = torch.empty(2 * n + 16, dtype=sdt, device=DEV)
            d.out, d.out2 = buf[:n], buf[n:2 * n]          # for odd n the second half is misaligned
            cuda_backend.set_tuning(variant, 0, 0)
            m, o = cuda_backend.step(d)
            cuda_backend.set_tuning(2, 0, 0)
            assert o.data_ptr() == buf.data_ptr()
            assert torch.equal(buf[:n].cpu(), ref_o) and torch.equal(buf[n:2 * n].cpu(), ref_o) and torch.equal(m.cpu(), ref_m)


def test_channels_last_layout_is_kept(cuda_backend):
    """Dense channels_last operands are used in place (no NCHW copy) and the outputs keep the layout."""
    g = torch.Generator(device=DEV).manual_seed(4)
    mk = lambda: torch.randn(6, 4, 32, 32, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    x, ec, eu, m1 = mk(), mk(), mk(), mk()
    a = StepArgs(form=FORM_DIFF2, n_model=2, x=x, xe=x, e_cond=ec, e_uncond=eu, m1=m1, predict_x0=True, guidance=7.5,
                 alpha_e=0.8, sigma_e=0.6, want_m_out=True, **coeffs(FORM_DIFF2, 3))
    before = cuda_backend.launch_count()
    m, o = cuda_backend.step(a)
    assert cuda_backend.launch_count() - before == 1
    assert m.is_contiguous(memory_format=torch.channels_last) and o.is_contiguous(memory_format=torch.channels_last)
    ref_m, ref_o = OracleBackend().step(StepArgs(**{**a.__dict__, "x": x.cpu(), "xe": x.cpu(), "e_cond": ec.cpu(), "e_uncond": eu.cpu(), "m1": m1.cpu()}))
    assert torch.equal(m.cpu(), ref_m) and torch.equal(o.cpu(), ref_o)
    # mixed layouts still give the right values (inputs are brought to one layout)
    a.m1 = m1.contiguous()
    m2, o2 = cuda_backend.step(a)
    assert torch.equal(o2, o) and torch.equal(m2, m)


def test_sample_with_channels_last_network(golden, cuda_backend):
    from cases import exact_net, seeded
    from dpm_solver_b200 import DPM_Solver, model_wrapper
    from helpers import product_schedule
    ns = product_schedule("sd")
    net = lambda xx, tt: exact_net(xx, tt).contiguous(memory_format=torch.channels_last)
    s = DPM_Solver(model_wrapper(net, ns), ns)
    x = seeded((2, 4, 16, 16), 1234).cuda().contiguous(memory_format=torch.channels_last)
    y = s.sample(x, steps=20, order=2)
    assert y.is_contiguous(memory_format=torch.channels_last)
    np.testing.assert_array_equal(y.cpu().numpy(), golden["samples"]["pp2m/y"])


@pytest.mark.parametrize("sdt", [torch.float32, torch.bfloat16, torch.float16])
def test_duplicate_equals_cat(cuda_backend, sdt):
    """dpm_duplicate == torch.cat([x] * 2) (model_wrapper :326): tile-multiple, ragged, tiny, unaligned view, NaN/inf
    payloads (a pure byte copy), channels_last."""
    for shape in [(64, 4, 64, 64), (3, 4, 33, 17), (1, 1, 1, 8), (5, 3, 7, 7), (2, 1, 1, 1)]:
        x = torch.randn(shape, device=DEV).to(sdt)
        x.view(-1)[0] = float("nan")
        x.view(-1)[-1] = float("inf")
        got = cuda_backend.duplicate(x)
        want = torch.cat([x] * 2)
        assert got.shape == want.shape and got.dtype == want.dtype
        assert torch.equal(got.view(torch.int16 if sdt != torch.float32 else torch.int32),
                           want.view(torch.int16 if sdt != torch.float32 else torch.int32))
    base = torch.randn(2 * 4 * 9 * 9 + 1, device=DEV).to(sdt)
    v = base[1:].view(2, 4, 9, 9)                                  # misaligned view -> copy fallback
    assert torch.equal(cuda_backend.duplicate(v), torch.cat([v] * 2))
    xc = torch.randn(4, 8, 16, 16, device=DEV).to(sdt).contiguous(memory_format=torch.channels_last)
    got = cuda_backend.duplicate(xc)
    assert got.is_contiguous(memory_format=torch.channels_last) and torch.equal(got, torch.cat([xc] * 2))
