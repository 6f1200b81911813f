"""Multi-condition classifier-free guidance (`model_wrapper(..., condition=[c1, ..., cK], guidance_scale=[s1, ..., sK])`)
on the CPU: the product's host logic, driven by a numpy executor that applies the K-term combine, against the UNMODIFIED
reference composed the way a user would compose it: each term from the reference's own model_wrapper for its condition
at guidance_scale=1 (the converted conditional output), combined left to right in eager fp32 torch, and the reference
DPM_Solver run on that as a noise model."""
import dataclasses
from unittest import mock

import numpy as np
import pytest
import torch

from cases import seeded
from oracle_backend import OracleBackend, _np
from test_cfg_rescale import inner_net, schedules

f32 = np.float32
B = 3
SHAPE = (B, 2, 4, 4)
# negative and zero scales; every value is an fp32 number, so the reference's python floats round to the same scales
SCALES = {2: [7.5, -2.0], 3: [4.0, 0.0, -1.5], 4: [3.0, 1.0, -0.5, 0.0]}


class MultiOracle(OracleBackend):
    """OracleBackend plus the multi-condition step (StepArgs.e_conds / scales / replicas) and `replicate`: every block
    converted by the parameterisation, then eps = eps_u; eps = eps + s_k*(eps_k - eps_u) in fp32 numpy."""

    def replicate(self, x, copies):
        self.launches += 1
        self.log.append(("replicate", copies))
        return torch.cat([x] * copies)

    def step(self, a):
        if a.e_conds is not None:
            self.log.append(("multi", a.form))
        m, o = super().step(a)
        if a.replicas is not None and o is not None:
            for r in a.replicas:
                r.copy_(o.reshape(r.shape))
        return m, o

    def _model_value(self, a, thr=None):
        if a.e_conds is None:
            return super()._model_value(a, thr)
        xe = _np(a.xe if a.xe is not None else a.x)
        with np.errstate(all="ignore"):
            eu = self._convert(a, _np(a.e_uncond), xe).astype(f32)
            eps = eu
            for s, e in zip(a.scales, a.e_conds):
                eps = (eps + f32(s) * (self._convert(a, _np(e), xe) - eu)).astype(f32)
        one = dataclasses.replace(a, n_model=1, param=0, e_cond=torch.from_numpy(eps), e_uncond=None, e_conds=None,
                                  scales=None)
        return super()._model_value(one, thr)


@pytest.fixture()
def multi_backend():
    from dpm_solver_b200 import ops
    be = MultiOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def conds(K, batch=B):
    return [torch.full((batch, 1), float(k + 1)) for k in range(K)]


def _kw(algo, thr):
    return dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)


def product_fn(model_type, K, scales, net=None, batch=B, **wkw):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    return new.model_wrapper(net or inner_net(), pns, model_type=model_type, guidance_type="classifier-free",
                             condition=conds(K, batch), unconditional_condition=torch.zeros(batch, 1),
                             guidance_scale=scales, **wkw), pns


def product(model_type, algo, thr, K, scales, **skw):
    import dpm_solver_b200 as new
    fn, pns = product_fn(model_type, K, scales)
    return new.DPM_Solver(fn, pns, **_kw(algo, thr), **skw)


def reference_composed(model_type, K, scales, batch=B):
    """model_fn(x, t_continuous) of the reference composition."""
    ref, rns, _ = schedules("sd")
    uc = torch.zeros(batch, 1)
    fs = [ref.model_wrapper(inner_net(), rns, model_type=model_type, guidance_type="classifier-free", condition=c,
                            unconditional_condition=uc, guidance_scale=1.0) for c in [uc] + conds(K, batch)]

    def composed(x, t):
        eu = fs[0](x, t)
        e = eu
        for s, f in zip(scales, fs[1:]):
            e = e + s * (f(x, t) - eu)
        return e
    return ref, rns, composed


def reference(model_type, algo, thr, K, scales):
    ref, rns, composed = reference_composed(model_type, K, scales)
    return ref.DPM_Solver(composed, rns, **_kw(algo, thr))


FIXED = [("multistep", 2), ("multistep", 3), ("singlestep", 3), ("singlestep_fixed", 2)]
ALGOS = [("dpmsolver", False), ("dpmsolver", True), ("dpmsolver++", False), ("dpmsolver++", True)]
MODELS = ["noise", "x_start", "v", "score"]


@pytest.mark.parametrize("K", [2, 3, 4])
@pytest.mark.parametrize("algo,thr", ALGOS)
@pytest.mark.parametrize("method,order", FIXED)
@pytest.mark.parametrize("model_type", MODELS)
def test_sample_matches_reference_composition(multi_backend, model_type, method, order, algo, thr, K):
    x = seeded(SHAPE, 11)
    kw = dict(steps=6, order=order, method=method, skip_type="time_uniform",
              denoise_to_zero=model_type in ("noise", "v"), return_intermediate=True)
    yp, ip = product(model_type, algo, thr, K, SCALES[K]).sample(x.clone(), **kw)
    yr, ir = reference(model_type, algo, thr, K, SCALES[K]).sample(x.clone(), **kw)
    np.testing.assert_array_equal(yp.numpy(), yr.numpy())
    assert len(ip) == len(ir)
    for a, b in zip(ip, ir):
        np.testing.assert_array_equal(a.numpy(), b.numpy())
    assert any(e[0] == "multi" for e in multi_backend.log)


def _adaptive(solver, x, order):
    with mock.patch("builtins.print") as pr:
        y = solver.sample(x.clone(), order=order, method="adaptive", atol=0.05, rtol=0.1)
        return y, pr.call_args[0][-1]


@pytest.mark.parametrize("order", [2, 3])
@pytest.mark.parametrize("algo,thr", ALGOS)
@pytest.mark.parametrize("model_type,K", [("noise", 2), ("x_start", 3), ("v", 4), ("score", 2)])
def test_adaptive_matches_reference_composition(multi_backend, model_type, K, algo, thr, order):
    """The host controller: the same NFE, and the result within the reduction-order tolerance of its error estimate
    (as for one condition)."""
    x = seeded(SHAPE, 11)
    yr, nfe_r = _adaptive(reference(model_type, algo, thr, K, SCALES[K]), x, order)
    yp, nfe_p = _adaptive(product(model_type, algo, thr, K, SCALES[K]), x, order)
    assert nfe_p == nfe_r
    err = np.abs(yp.numpy().astype(np.float64) - yr.numpy()).max() / max(np.abs(yr.numpy()).max(), 1e-30)
    assert err <= 1e-5


def _run_logged(be, model_type, cond, scale, thr):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    fn = new.model_wrapper(inner_net(), pns, model_type=model_type, guidance_type="classifier-free", condition=cond,
                           unconditional_condition=torch.zeros(B, 1), guidance_scale=scale)
    be.log.clear()
    n0 = be.launches
    y = new.DPM_Solver(fn, pns, **_kw("dpmsolver++", thr)).sample(seeded(SHAPE, 5), steps=5, order=2)
    return y, be.launches - n0, list(be.log)


@pytest.mark.parametrize("thr", [False, True])
@pytest.mark.parametrize("model_type", ["noise", "v"])
@pytest.mark.parametrize("scale", [7.5, 1.0, -2.0])
def test_one_condition_in_a_list_is_the_tensor_form(multi_backend, model_type, scale, thr):
    c = torch.ones(B, 1)
    y_list, n_list, log_list = _run_logged(multi_backend, model_type, [c], [scale], thr)
    y_one, n_one, log_one = _run_logged(multi_backend, model_type, c, scale, thr)
    assert (n_list, log_list) == (n_one, log_one)
    assert not any(e[0] in ("multi", "replicate") for e in log_list)
    np.testing.assert_array_equal(y_list.numpy(), y_one.numpy())


@pytest.mark.parametrize("thr", [False, True])
@pytest.mark.parametrize("K", [2, 4])
def test_launches_and_network_calls(multi_backend, K, thr):
    """One network call per evaluation on (K+1)B rows with the conditions in the order [uc, c1, ..., cK]; one fused
    launch per evaluation, plus the materialising launch and the quantile with thresholding; the first network input
    from one replicate launch, the later ones written by the fused steps."""
    import dpm_solver_b200 as new
    calls = []
    inner = inner_net()

    def net(x, t, c):
        calls.append((tuple(x.shape), c[:, 0].tolist()))
        return inner(x, t, c)
    fn, pns = product_fn("noise", K, SCALES[K], net=net)
    nfe = 5
    multi_backend.log.clear()
    n0 = multi_backend.launches
    new.DPM_Solver(fn, pns, **_kw("dpmsolver++", thr)).sample(seeded(SHAPE, 5), steps=nfe, order=2)
    log = list(multi_backend.log)
    assert len(calls) == nfe
    for shape, c in calls:
        assert shape == ((K + 1) * B,) + SHAPE[1:]
        assert c == [float(k) for k in range(K + 1) for _ in range(B)]
    assert log.count(("replicate", K + 1)) == 1
    fused = [e for e in log if e[0] == "multi" and e[1] != 0]
    assert len(fused) == nfe
    if thr:
        # the materialised noise (FORM_NONE) feeds the quantile; the fused step recomputes the combine
        assert log.count(("multi", 0)) == nfe and log.count(("quantile", 1)) == nfe
        assert multi_backend.launches - n0 == 1 + 3 * nfe
    else:
        assert ("multi", 0) not in log
        assert multi_backend.launches - n0 == 1 + nfe


@pytest.mark.parametrize("K", [2, 3, 4])
def test_direct_model_fn_call(multi_backend, K):
    """model_fn(x, t) is the combined noise, for one time label and for one label per sample."""
    x = seeded(SHAPE, 3)
    for model_type in MODELS:
        fn, _ = product_fn(model_type, K, SCALES[K])
        _, _, composed = reference_composed(model_type, K, SCALES[K])
        for t in (torch.full((B,), 0.6), torch.linspace(0.9, 0.2, B)):
            np.testing.assert_array_equal(fn(x, t).numpy(), composed(x, t).numpy())


def test_invalid_arguments_raise(multi_backend):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    calls = []
    net = inner_net(calls)
    uc = torch.zeros(B, 1)
    mk = lambda cond, scale, **kw: new.model_wrapper(net, pns, guidance_type="classifier-free", condition=cond,
                                                     unconditional_condition=kw.pop("uc", uc), guidance_scale=scale,
                                                     **kw)
    cases = [
        (conds(5), [1.0] * 5, {}, "1 to 4"),                                 # more than four conditions
        (conds(3), [1.0, 2.0], {}, "2 guidance scales for 3"),               # a count other than K
        (conds(2), 7.5, {}, "single scale"),                                  # a scalar scale with a list
        (conds(2), torch.tensor(7.5), {}, "single scale"),
        (conds(2), [1.0, 2.0], dict(uc=None), "unconditional_condition"),
        (conds(2), [1.0, 2.0], dict(guidance_rescale=0.7), "guidance_rescale"),
        (conds(2), torch.ones(B, 2), {}, "per-sample"),                       # per-sample x per-condition scales
    ]
    for cond, scale, kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            mk(cond, scale, **kw)
    with pytest.raises(ValueError, match="reference_rounding"):
        new.DPM_Solver(mk(conds(2), [1.0, 2.0]), pns, algorithm_type="dpmsolver", reference_rounding=True)
    assert calls == []


def test_scales_are_read_once_and_rounded_to_fp32(multi_backend):
    s = torch.tensor([0.1, 3.0], dtype=torch.float64)
    fn, _ = product_fn("noise", 2, s)
    assert fn.cond_scales == (float(np.float32(0.1)), 3.0)
    s[0] = 5.0                       # read on the host once, in model_wrapper
    assert fn.cond_scales[0] == float(np.float32(0.1))
    fn2, _ = product_fn("noise", 2, (0.1, 3.0))
    assert fn2.cond_scales == fn.cond_scales


def test_sequence_condition_outside_cfg_is_untouched(multi_backend):
    """Only classifier-free guidance reads a list of conditions as several conditions."""
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    cond = [torch.ones(B, 1)]
    fn = new.model_wrapper(lambda x, t: x * 0.5, pns, guidance_type="uncond", condition=cond, guidance_scale=[1.0, 2.0])
    assert fn.n_cond == 0 and fn.condition is cond and fn.input_rows(B) == B
