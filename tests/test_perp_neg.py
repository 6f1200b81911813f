"""Perp-Neg (`model_wrapper(..., condition=[c_pos, c_neg, ...], perp_neg=True)`) on the CPU: the product's host logic
on the numpy executor (tests/perpneg_oracle.py). The words against a float64 transcription of the formula and against
exactly rounded sums; sample() bit for bit against the UNMODIFIED reference composed the way a user would compose it
(each block from the reference's own model_wrapper at guidance_scale=1, the words from the raw outputs, the combine in
eager fp32 torch); the identities, rows, launch counts, batch sharding and the rejections."""
import os

import numpy as np
import pytest
import torch

from oracle import ref_loader
from perpneg_oracle import (NAN32, PerpNegOracle, fold_order_case, guided_net, perp_combine, perpneg_reference,
                            sums_exact, words_exact, words_final, words_final_reversed, words_fsum)

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="no reference checkout and no oracle/_ref")
f32 = np.float32
B, SHAPE = 2, (2, 3, 6, 6)
SCALES = {2: [7.5, -3.0], 3: [5.0, -2.0, -1.5], 4: [4.0, -1.0, -0.5, -2.5]}
MODEL_TYPES = ["noise", "x_start", "v", "score", "flow", "edm"]
VP_TYPES = ["noise", "x_start", "v", "score"]


@pytest.fixture()
def pn_backend():
    from dpm_solver_b200 import ops
    be = PerpNegOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def net(x, t, c):
    """A time-independent network whose conditional directions differ nonlinearly from each other (no d_k is a multiple
    of d_1); uc = 0 gives the unconditional output."""
    cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x + 0.25 * cc * torch.cos(0.7 * x + cc) - 0.1


def blind(x, t, c):
    return 0.5 * torch.sin(1.3 * x) + 0.4 * x - 0.1


def counted(calls, model=net):
    def f(x, t, c):
        calls.append(tuple(x.shape))
        return model(x, t, c)
    return f


def conds(K, batch=B):
    return [torch.full((batch, 1), float(k + 1)) for k in range(K)]


def product_schedule(mt):
    import dpm_solver_b200 as new
    from helpers import product_schedule as vp
    if mt == "flow":
        return new.NoiseScheduleFlow(shift=3.0)
    if mt == "edm":
        return new.NoiseScheduleEDM()
    return vp("sd")


def wrap(mt, ns, K=2, model=net, batch=B, scales=None, **kw):
    import dpm_solver_b200 as new
    return new.model_wrapper(model, ns, model_type=mt, guidance_type="classifier-free", condition=conds(K, batch),
                             unconditional_condition=torch.zeros(batch, 1),
                             guidance_scale=SCALES[K] if scales is None else scales, **kw)


def reference_composed(mt, K, model=net, batch=B, scales=None, rns=None, condition=None):
    """(ref module, ref schedule, model_fn) of the reference composition: each block from the reference's model_wrapper
    for its condition at scale 1 (converted to noise), the words from the raw outputs those calls made, then
    eps_u + w_1*(eps_1 - eps_u) + s_2*(eps_2 - eps_u) + ... in eager fp32 torch. `scales` (default SCALES[K]), the
    reference VP schedule `rns` (default "sd") and the K conditions `condition` (default conds(K, batch)) may be given;
    the words read the raw outputs row-major, so the network must return row-major outputs."""
    from test_cfg_rescale import schedules
    ref, sd_rns, _ = schedules("sd")
    rns = sd_rns if rns is None else rns
    uc = torch.zeros(batch, 1)
    raw = []

    def recorded(x, t, c):
        out = model(x, t, c)
        raw.append(out)
        return out
    fs = [ref.model_wrapper(recorded, rns, model_type=mt, guidance_type="classifier-free", condition=c,
                            unconditional_condition=uc, guidance_scale=1.0)
          for c in [uc] + (conds(K, batch) if condition is None else list(condition))]
    scales = SCALES[K] if scales is None else list(scales)

    def composed(x, t):
        raw.clear()
        eps = [f(x, t) for f in fs]
        w1 = words_exact(raw[0].reshape(batch, -1).numpy(), [r.reshape(batch, -1).numpy() for r in raw[1:]], scales)
        return perp_combine(eps[0], eps[1:], scales, torch.from_numpy(w1))
    return ref, rns, composed


def x_T(seed=0, batch=B):
    return torch.randn((batch,) + SHAPE[1:], generator=torch.Generator().manual_seed(seed))


def ulps(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


# ---- the words -------------------------------------------------------------------------------------------------------

def _draws(seed, n=200):
    """Seeded (u, e_1..e_K, scales) draws of varied size, angle and norm."""
    rng = np.random.default_rng(seed)
    for _ in range(n):
        K = int(rng.integers(2, 5))
        D = int(rng.integers(2, 300))
        u = (rng.standard_normal((1, D)) * 10.0 ** rng.uniform(-1, 1)).astype(f32)
        d1 = rng.standard_normal((1, D)) * 10.0 ** rng.uniform(-2, 1)
        es = [(u + d1).astype(f32)]
        for _ in range(K - 1):
            dk = rng.uniform(-1, 1) * d1 + rng.standard_normal((1, D)) * 10.0 ** rng.uniform(-2, 1)
            es.append((u + dk).astype(f32))
        scales = [float(f32(v)) for v in [rng.uniform(1, 10)] + list(-rng.uniform(0, 5, K - 1))]
        yield u, es, scales


def test_executor_words_match_the_formula():
    """The executor's fold, before its final fp32 rounding, gives eps within 1e-12 (relative) of the float64
    transcription of the formula."""
    worst = 0.0
    for u, es, s in _draws(5):
        N, P = sums_exact(u, es)
        w64 = float(s[0])
        for sk, pk in zip(s[1:], P):
            w64 = w64 - sk * (float(pk[0]) / float(N[0]))
        u64 = u.astype(np.float64)
        d = [e.astype(np.float64) - u64 for e in es]
        got = u64 + w64 * d[0]
        for sk, dk in zip(s[1:], d[1:]):
            got = got + sk * dk
        want = perpneg_reference(u, es, s)
        worst = max(worst, float(np.abs(got - want).max() / np.abs(want).max()))
        assert words_exact(u, es, s)[0] == f32(w64)
    assert worst <= 1e-12, worst


@pytest.mark.parametrize("per_sample", [7, 8, 9, 8192 + 16, 8193, 3 * 64 * 64])
@pytest.mark.parametrize("K", [2, 3, 4])
def test_words_within_the_final_rounding_of_fsum(per_sample, K):
    rng = np.random.default_rng(per_sample + K)
    u = rng.standard_normal((3, per_sample)).astype(f32)
    es = [(u + rng.standard_normal((3, per_sample)) * (0.3 + k)).astype(f32) for k in range(K)]
    es[1][2] = (u[2] + 0.5 * (es[0][2] - u[2]) + 1e-3 * rng.standard_normal(per_sample)).astype(f32)
    got, want = words_exact(u, es, SCALES[K]), words_fsum(u, es, SCALES[K])
    assert ulps(got, want).max() <= 1, (got, want)


def test_words_read_each_sample_alone():
    rng = np.random.default_rng(1)
    u = rng.standard_normal((4, 8193)).astype(f32)
    es = [rng.standard_normal((4, 8193)).astype(f32) for _ in range(3)]
    full = words_exact(u, es, SCALES[3])
    for b in range(4):
        assert words_exact(u[b:b + 1], [e[b:b + 1] for e in es], SCALES[3])[0] == full[b]


def test_constructed_words():
    rng = np.random.default_rng(3)
    D = 64
    u = rng.standard_normal((1, D)).astype(f32)
    s = SCALES[2]
    # d_2 _|_ d_1 on disjoint elements: w_1 == s_1 exactly
    e1, e2 = u.copy(), u.copy()
    e1[0, :10] += 1.0
    e2[0, 10:20] -= 2.0
    assert words_exact(u, [e1, e2], s)[0] == f32(s[0])
    # N == 0 (condition 1 equals u): c_2 = 0, w_1 == s_1
    assert words_exact(u, [u.copy(), e2], s)[0] == f32(s[0])
    # d_2 = 2*d_1 exactly: c_2 = 2, w_1 = s_1 - 2*s_2 (u on a grid of 1/16, so both sums are exact in fp32)
    u = (rng.integers(-64, 64, (1, D)) / 16).astype(f32)
    e1 = (u + 0.25).astype(f32)
    e2 = (u + 0.5).astype(f32)
    d1 = e1.astype(np.float64) - u
    assert np.array_equal(e2.astype(np.float64) - u, 2 * d1)
    assert words_exact(u, [e1, e2], s)[0] == f32(s[0] - s[1] * 2.0)
    # an inf or NaN output: the device's NaN
    for bad in (np.inf, -np.inf, np.nan):
        for which in range(3):
            blocks = [u.copy(), e1.copy(), e2.copy()]
            blocks[which][0, 5] = bad
            w = words_exact(blocks[0], blocks[1:], s)
            assert w.view(np.uint32)[0] == NAN32.view(np.uint32)
    # the fold itself: left to right, each op rounded
    assert words_final([4.0], [[2.0], [-8.0]], [3.0, -1.0, 0.5])[0] == f32((3.0 - (-1.0) * 0.5) - 0.5 * (-2.0))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_fold_order_case_tells_the_orders_apart(seed):
    """fold_order_case's words are exact where they should be (c_2 = 2^13, c_4 = -2^13) and differ in several samples
    from the words of the reversed fold, so a device test on them fails for a kernel that folds in another order."""
    u, es, s = fold_order_case(seed=seed)
    N, P = sums_exact(u, es)
    assert np.array_equal(P[0] / N, np.full(len(N), 8192.0)) and np.array_equal(P[2] / N, np.full(len(N), -8192.0))
    w = words_exact(u, es, s)
    assert np.array_equal(w, words_final(N, P, s))
    assert (w != words_final_reversed(N, P, s)).sum() >= 2


# ---- sample() against the reference ----------------------------------------------------------------------------------

METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 1), ("singlestep", 2),
           ("singlestep", 3), ("singlestep_fixed", 2)]
ALGOS = [("dpmsolver", False), ("dpmsolver++", False), ("dpmsolver++", True)]


def _solver_kw(algo, thr):
    return dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)


@needs_ref
@pytest.mark.parametrize("K", [2, 3, 4])
@pytest.mark.parametrize("algo,thr", ALGOS)
@pytest.mark.parametrize("method,order", METHODS)
@pytest.mark.parametrize("mt", VP_TYPES)
def test_sample_matches_reference_composition(pn_backend, mt, method, order, algo, thr, K):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    kw = dict(steps=6, order=order, method=method, skip_type="time_uniform")
    y = new.DPM_Solver(wrap(mt, ns, K, perp_neg=True), ns, **_solver_kw(algo, thr)).sample(x_T(), **kw)
    ref, rns, composed = reference_composed(mt, K)
    yr = ref.DPM_Solver(composed, rns, **_solver_kw(algo, thr)).sample(x_T(), **kw)
    assert torch.equal(y, yr), float((y - yr).abs().max())


@needs_ref
@pytest.mark.parametrize("mt", ["noise", "v", "score"])
@pytest.mark.parametrize("algo,thr", ALGOS)
def test_adaptive_host_controller_matches_reference(pn_backend, mt, algo, thr, capsys):
    """The same evaluations and the result within 1e-5. (x_start is left out: its eps = (x - alpha*x0)/sigma divides by
    a small sigma_t near the end, so rounding-level differences of the controller's scalars flip a step decision; its
    fixed-grid runs above are bit-identical.)"""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    kw = dict(order=2, method="adaptive", atol=0.0078, rtol=0.05)
    calls = []
    y = new.DPM_Solver(wrap(mt, ns, 2, model=counted(calls), perp_neg=True), ns, **_solver_kw(algo, thr)).sample(
        x_T(), **kw)
    ref_calls = []
    ref, rns, composed = reference_composed(mt, 2, model=counted(ref_calls))
    yr = ref.DPM_Solver(composed, rns, **_solver_kw(algo, thr)).sample(x_T(), **kw)
    capsys.readouterr()
    assert len(calls) * 3 == len(ref_calls)           # one (K+1)-fold call against K+1 single calls per evaluation
    err = float((y.double() - yr.double()).abs().max() / yr.double().abs().max())
    assert err <= 1e-5, err


@needs_ref
@pytest.mark.parametrize("mt", VP_TYPES)
@pytest.mark.parametrize("algo", ["dpmsolver", "dpmsolver++"])
def test_denoise_to_zero_inverse_and_intermediates_match_reference(pn_backend, mt, algo):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    ref, rns, composed = reference_composed(mt, 3)
    skw = dict(steps=6, order=2, method="multistep", denoise_to_zero=True)
    y = new.DPM_Solver(wrap(mt, ns, 3, perp_neg=True), ns, algorithm_type=algo).sample(x_T(), **skw)
    assert torch.equal(y, ref.DPM_Solver(composed, rns, algorithm_type=algo).sample(x_T(), **skw))
    ikw = dict(steps=5, order=2, method="multistep")
    yi = new.DPM_Solver(wrap(mt, ns, 3, perp_neg=True), ns, algorithm_type=algo).inverse(x_T(1), **ikw)
    assert torch.equal(yi, ref.DPM_Solver(composed, rns, algorithm_type=algo).inverse(x_T(1), **ikw))
    # return_intermediate with both hooks
    hx0 = lambda x0, t: x0 * 0.9
    hxt = lambda x, t, step: x * 0.99
    kw = dict(steps=5, order=2, method="multistep", return_intermediate=True)
    got = new.DPM_Solver(wrap(mt, ns, 3, perp_neg=True), ns, algorithm_type=algo, correcting_x0_fn=hx0,
                         correcting_xt_fn=hxt).sample(x_T(2), **kw)
    want = ref.DPM_Solver(composed, rns, algorithm_type=algo, correcting_x0_fn=hx0,
                          correcting_xt_fn=hxt).sample(x_T(2), **kw)
    assert torch.equal(got[0], want[0]) and len(got[1]) == len(want[1])
    assert all(torch.equal(a, b) for a, b in zip(got[1], want[1]))


@needs_ref
def test_noise_network_matches_the_reference_uncond_wrapper(pn_backend):
    """guided_net: the unmodified reference's guidance_type="uncond" wrapper on the Perp-Neg noise."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    ref, rns, _ = reference_composed("noise", 2)
    g = guided_net(net, torch.zeros(B, 1), conds(2), SCALES[2])
    kw = dict(steps=6, order=3, method="multistep")
    y = new.DPM_Solver(wrap("noise", ns, 2, perp_neg=True), ns).sample(x_T(), **kw)
    assert torch.equal(y, ref.DPM_Solver(ref.model_wrapper(g, rns), rns).sample(x_T(), **kw))


# ---- every model type: the masked path with the words -------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("algo,thr", ALGOS)
@pytest.mark.parametrize("method,order", [("multistep", 3), ("singlestep", 2), ("adaptive", 2)])
def test_every_model_type_is_the_masked_run_on_its_words(pn_backend, mt, algo, thr, method, order, capsys):
    """A Perp-Neg run equals the regional-guidance run with scales (1, s_2, ...) whose [B, 1, 1, 1] mask of condition 1
    the network rewrites in place with the words of its own outputs at every call."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    K, s = 3, SCALES[3]
    mask = torch.ones(B, 1, 1, 1)

    def hooked(x, t, c):
        out = net(x, t, c)
        o = out.chunk(K + 1)
        w = words_exact(o[0].reshape(B, -1).numpy(), [e.reshape(B, -1).numpy() for e in o[1:]], s)
        mask.copy_(torch.from_numpy(w).reshape(B, 1, 1, 1))
        return out
    kw = dict(steps=6, order=order, method=method) if method != "adaptive" else dict(order=2, method=method,
                                                                                    atol=0.05, rtol=0.1)
    y = new.DPM_Solver(wrap(mt, ns, K, perp_neg=True), ns, **_solver_kw(algo, thr)).sample(x_T(), **kw)
    ym = new.DPM_Solver(wrap(mt, ns, K, model=hooked, scales=[1.0] + s[1:], guidance_mask=[mask, None, None]), ns,
                        **_solver_kw(algo, thr)).sample(x_T(), **kw)
    capsys.readouterr()
    assert torch.equal(y, ym)


@pytest.mark.parametrize("mt", MODEL_TYPES)
def test_direct_model_fn_call(pn_backend, mt):
    """model_fn(x, t) is the masked combine with the words, per-sample time labels included."""
    ns = product_schedule(mt)
    fn = wrap(mt, ns, 2, perp_neg=True)
    x = x_T(3)
    for t in (torch.full((B,), 0.5), torch.tensor([0.5, 0.3])):
        o = net(torch.cat([x] * 3), None, torch.cat([torch.zeros(B, 1)] + conds(2))).chunk(3)
        w = words_exact(o[0].reshape(B, -1).numpy(), [e.reshape(B, -1).numpy() for e in o[1:]], SCALES[2])
        want = wrap(mt, ns, 2, scales=[1.0, SCALES[2][1]], guidance_mask=[torch.from_numpy(w).reshape(B, 1, 1, 1),
                                                                          None])(x, t)
        assert torch.equal(fn(x, t), want)


# ---- identities, rows, counts, sharding ------------------------------------------------------------------------------

@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("thr", [False, True])
def test_perpendicular_negatives_leave_the_run_unchanged(pn_backend, mt, thr):
    """Conditions that differ from u on disjoint elements: the words are s_1, and the run is the run without perp_neg."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)

    def disjoint(x, t, c):
        cc = c.reshape(-1, 1, 1, 1)
        sel = torch.zeros_like(x)
        sel[:, :, :3] = (cc == 1).float()          # condition 1 on rows 0..2
        sel[:, :, 3:] = (cc == 2).float() * 2      # condition 2 on rows 3..5
        return blind(x, t, c) + sel * torch.cos(0.7 * x)
    pn_backend.log.clear()
    kw = dict(algorithm_type="dpmsolver++", correcting_x0_fn="dynamic_thresholding" if thr else None)
    y = new.DPM_Solver(wrap(mt, ns, 2, model=disjoint, perp_neg=True), ns, **kw).sample(x_T(), steps=6, order=2)
    y0 = new.DPM_Solver(wrap(mt, ns, 2, model=disjoint), ns, **kw).sample(x_T(), steps=6, order=2)
    assert torch.equal(y, y0)


@pytest.mark.parametrize("mt", MODEL_TYPES)
@pytest.mark.parametrize("state_dtype", [None, torch.bfloat16])
def test_condition_blind_run_equals_the_unguided_run(pn_backend, mt, state_dtype):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    kw = dict(steps=6, order=2)
    y = new.DPM_Solver(wrap(mt, ns, 3, model=blind, perp_neg=True), ns, state_dtype=state_dtype).sample(x_T(), **kw)
    y0 = new.DPM_Solver(new.model_wrapper(lambda x, t: blind(x, t, None), ns, model_type=mt), ns,
                        state_dtype=state_dtype).sample(x_T(), **kw)
    assert torch.equal(y, y0)


@pytest.mark.parametrize("mt", ["noise", "v", "flow"])
def test_parallel_negative_vanishes(pn_backend, mt):
    """d_2 = 2*d_1 exactly: the negative's effect is removed, leaving one-condition CFG with s_1, to rounding."""
    import dpm_solver_b200 as new
    ns = product_schedule(mt)

    def parallel(x, t, c):
        cc = c.reshape(-1, 1, 1, 1)
        return blind(x, t, c) + cc * 0.25          # d_k = 0.25*c_k, exact in fp32
    y = new.DPM_Solver(wrap(mt, ns, 2, model=parallel, perp_neg=True), ns).sample(x_T(), steps=6, order=2)
    y1 = new.DPM_Solver(new.model_wrapper(parallel, ns, model_type=mt, guidance_type="classifier-free",
                                          condition=conds(1)[0], unconditional_condition=torch.zeros(B, 1),
                                          guidance_scale=SCALES[2][0]), ns).sample(x_T(), steps=6, order=2)
    y_plain = new.DPM_Solver(wrap(mt, ns, 2, model=parallel), ns).sample(x_T(), steps=6, order=2)
    err = float((y - y1).abs().max() / y1.abs().max())
    assert err <= 1e-5, err
    assert float((y_plain - y1).abs().max() / y1.abs().max()) > 1e-2      # without perp_neg the negative acts


@pytest.mark.parametrize("mt", ["noise", "x_start", "flow", "edm"])
def test_each_row_equals_its_single_sample_run(pn_backend, mt):
    import dpm_solver_b200 as new
    ns = product_schedule(mt)
    x = x_T(4, batch=3)
    c3 = [torch.tensor([[1.0], [2.5], [0.5]]), torch.tensor([[2.0], [3.0], [-1.0]])]

    def run(rows):
        fn = new.model_wrapper(net, ns, model_type=mt, guidance_type="classifier-free", condition=[c[rows] for c in c3],
                               unconditional_condition=torch.zeros(3, 1)[rows], guidance_scale=SCALES[2],
                               perp_neg=True)
        return new.DPM_Solver(fn, ns, correcting_x0_fn="dynamic_thresholding").sample(x[rows], steps=5, order=2)
    yb = run(slice(None))
    for b in range(3):
        assert torch.equal(yb[b:b + 1], run(slice(b, b + 1)))


@pytest.mark.parametrize("thr", [False, True])
def test_launch_and_network_call_counts(pn_backend, thr):
    """Per guided evaluation: the run without perp_neg plus the words pass (2 launches); one network call on (K+1)B
    rows."""
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    K = 3
    kw = dict(correcting_x0_fn="dynamic_thresholding" if thr else None)
    counts = []
    for perp in (False, True):
        calls = []
        s = new.DPM_Solver(wrap("noise", ns, K, model=counted(calls), perp_neg=perp), ns, **kw)
        pn_backend.log.clear()
        n0 = pn_backend.launch_count()
        s.sample(x_T(), steps=5, order=2)
        counts.append(pn_backend.launch_count() - n0)
        assert calls == [((K + 1) * B,) + SHAPE[1:]] * 5
        assert sum(e[0] == "perpneg_words" for e in pn_backend.log) == (5 if perp else 0)
    assert counts[1] - counts[0] == 2 * 5, counts


def test_two_sample_calls_and_a_fresh_solver_are_bit_identical(pn_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    fn = wrap("flow", ns, 2, perp_neg=True)
    s = new.DPM_Solver(fn, ns)
    y1, y2 = s.sample(x_T(), steps=5, order=2), s.sample(x_T(), steps=5, order=2)
    y3 = new.DPM_Solver(fn, ns).sample(x_T(), steps=5, order=2)
    assert torch.equal(y1, y2) and torch.equal(y1, y3)


def _sharded_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dpm_solver_b200 import ops
        import dpm_solver_b200 as new
        ops.set_backend(PerpNegOracle())
        ns = product_schedule("flow")
        x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))[2 * rank:2 * rank + 2]
        y = new.DPM_Solver(wrap("flow", ns, 2, perp_neg=True), ns, plan_broadcast=True).sample(x, steps=5, order=2)
        q.put((rank, y))
    finally:
        dist.destroy_process_group()


def test_batch_sharding_needs_no_collective(pn_backend):
    """Two gloo ranks of two samples each equal the unsharded run of four: the words are per sample."""
    import socket
    import torch.multiprocessing as mp
    import dpm_solver_b200 as new
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=300) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    ns = product_schedule("flow")
    x = torch.randn((4,) + SHAPE[1:], generator=torch.Generator().manual_seed(9))
    y = new.DPM_Solver(wrap("flow", ns, 2, batch=4, perp_neg=True), ns).sample(x, steps=5, order=2)
    assert torch.equal(torch.cat([got[0], got[1]]), y)


# ---- rejections ------------------------------------------------------------------------------------------------------

def _rejections(calls):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    uc, cs = torch.zeros(B, 1), conds(2)
    model = counted(calls)
    base = dict(guidance_type="classifier-free", condition=cs, unconditional_condition=uc, guidance_scale=SCALES[2])
    bad_wrap = [
        # Perp-Neg's own
        dict(base, perp_neg=1),
        dict(base, perp_neg="yes"),
        dict(guidance_type="uncond", perp_neg=True),
        dict(guidance_type="classifier", classifier_fn=lambda *a: None, condition=cs[0], perp_neg=True),
        dict(base, unconditional_condition=None, perp_neg=True),
        dict(base, condition=cs[0], guidance_scale=7.5, perp_neg=True),
        dict(base, condition=cs[:1], guidance_scale=[7.5], perp_neg=True),
        dict(base, guidance_mask=[torch.ones(6, 6), None], perp_neg=True),
        # what several conditions refuse
        dict(base, guidance_rescale=0.7, perp_neg=True),
        dict(base, guidance_scale=torch.ones(2, B), perp_neg=True),
        dict(base, apg_eta=0.0, perp_neg=True),
        dict(base, cfg_zero_star=True, perp_neg=True),
        dict(base, cfg_pp=True, perp_neg=True),
        dict(base, tcfg=True, perp_neg=True),
        dict(base, guidance_scale=1.0, fdg_scales=[2.0, 3.0], perp_neg=True),
    ]
    for kw in bad_wrap:
        yield lambda kw=kw: new.model_wrapper(model, ns, **kw)
    fn = new.model_wrapper(model, ns, perp_neg=True, **base)
    yield lambda: new.DPM_Solver(fn, ns, reference_rounding=True)
    yield lambda: new.UniPC(fn, ns).sample(x_T(), steps=5, order=2)


def test_rejections_launch_nothing(pn_backend):
    n, calls = 0, []
    for call in _rejections(calls):
        before = pn_backend.launch_count()
        with pytest.raises(ValueError):
            call()
        assert pn_backend.launch_count() == before and calls == []
        n += 1
    assert n == 17


def test_rejection_messages():
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    uc, cs = torch.zeros(B, 1), conds(2)
    base = dict(guidance_type="classifier-free", condition=cs, unconditional_condition=uc, guidance_scale=SCALES[2])
    for kw, msg in ((dict(base, perp_neg=1), "perp_neg must be a bool"),
                    (dict(base, unconditional_condition=None, perp_neg=True), "perp_neg needs guidance_type"),
                    (dict(base, condition=cs[0], guidance_scale=7.5, perp_neg=True), "at least two conditions"),
                    (dict(base, guidance_mask=[None, None], perp_neg=True), "perp_neg is not available with "
                                                                            "guidance_mask"),
                    (dict(base, guidance_rescale=0.5, perp_neg=True), "not available with several conditions"),
                    (dict(base, tcfg=True, perp_neg=True), "tcfg is not available with several conditions")):
        with pytest.raises(ValueError, match=msg):
            new.model_wrapper(net, ns, **kw)
