"""Per-sample classifier-free guidance (`model_wrapper(..., guidance_scale=scales[B])`) on the CPU: the product's host
logic, driven by a numpy executor that applies each sample's scale, against the UNMODIFIED reference run once per
distinct scale on the rows that carry it."""
import dataclasses
import os
from unittest import mock

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from cases import seeded
from oracle_backend import OracleBackend, _np
from test_cfg_rescale import PHI, inner_net, ratio64, ref_rescaled_net, schedules

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# 0, 1 (the bypass), negative and large scales; 7.5 twice
SCALES = [7.5, 1.0, 0.0, 7.5, -2.0, 60.0]
B = len(SCALES)
SHAPE = (B, 2, 4, 4)


class GuidedOracle(OracleBackend):
    """OracleBackend plus per-sample scales (StepArgs.guidance_b) and the guidance rescale: every sample is computed
    as the one-scale step with its own scale; a sample with scale 1 takes the conditional output alone."""

    def cfg_rescale_ratio(self, e_cond, e_uncond, guidance):
        self.launches += 2
        self.log.append(("ratio", 2))
        c, u = _np(e_cond), _np(e_uncond)
        s = _np(guidance).reshape((-1,) + (1,) * (c.ndim - 1)) if torch.is_tensor(guidance) else f32(guidance)
        with np.errstate(all="ignore"):
            g = (u + s * (c - u)).astype(f32)
        return torch.from_numpy(ratio64(c, g))

    def step(self, a):
        if a.guidance_b is not None:
            self.log.append(("guided", a.form))
        return super().step(a)

    def _one_scale(self, a, thr):
        if a.ratio is None:
            return super()._model_value(a, thr)
        c, u = _np(a.e_cond), _np(a.e_uncond)
        with np.errstate(all="ignore"):
            g = (u + f32(a.guidance) * (c - u)).astype(f32)
            r = np.repeat(_np(a.ratio), a.per_sample).reshape(g.shape)
            gp = (f32(a.phi) * (g * r) + f32(1.0 - a.phi) * g).astype(f32)
        return super()._model_value(dataclasses.replace(a, n_model=1, e_cond=torch.from_numpy(gp), e_uncond=None,
                                                        ratio=None), thr)

    def _model_value(self, a, thr=None):
        if a.guidance_b is None:
            return self._one_scale(a, thr)
        gb = _np(a.guidance_b)
        row = lambda t, b: None if t is None else t[b:b + 1]
        out = []
        for b in range(gb.size):
            ab = dataclasses.replace(a, e_cond=row(a.e_cond, b), e_uncond=row(a.e_uncond, b), x=row(a.x, b),
                                     xe=row(a.xe, b), ratio=row(a.ratio, b), guidance=float(gb[b]), guidance_b=None)
            if gb[b] == 1:      # the reference's bypass (:323)
                ab = dataclasses.replace(ab, n_model=1, e_uncond=None, ratio=None)
            out.append(self._one_scale(ab, None if thr is None else thr.reshape(-1)[b:b + 1]))
        return np.concatenate(out)


@pytest.fixture()
def guided_backend():
    from dpm_solver_b200 import ops
    be = GuidedOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def _kw(algo, thr):
    return dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thr else None)


def product(model_type, algo, thr, scales=SCALES, phi=0., batch=B, **wkw):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    fn = new.model_wrapper(inner_net(), pns, model_type=model_type, guidance_type="classifier-free",
                           condition=torch.ones(batch, 1), unconditional_condition=torch.zeros(batch, 1),
                           guidance_scale=scales, guidance_rescale=phi, **wkw)
    return new.DPM_Solver(fn, pns, **_kw(algo, thr))


def reference_rows(model_type, algo, thr, phi, run, x, scales=SCALES):
    """run(solver, x_rows) on the unmodified reference, once per distinct scale on the rows that carry it; returns
    [rows, result] pairs."""
    ref, rns, _ = schedules("sd")
    res = []
    for s in sorted(set(scales)):
        rows = [i for i, v in enumerate(scales) if v == s]
        uc, c = torch.zeros(len(rows), 1), torch.ones(len(rows), 1)
        if phi and s != 1:
            fn = ref.model_wrapper(ref_rescaled_net(inner_net(), uc, c, s, phi), rns, model_type=model_type)
        else:
            fn = ref.model_wrapper(inner_net(), rns, model_type=model_type, guidance_type="classifier-free",
                                   condition=c, unconditional_condition=uc, guidance_scale=s)
        res.append((rows, run(ref.DPM_Solver(fn, rns, **_kw(algo, thr)), x[rows].clone())))
    return res


FIXED = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 2), ("singlestep", 3),
         ("singlestep_fixed", 2)]
ALGOS = [("dpmsolver", False), ("dpmsolver", True), ("dpmsolver++", False), ("dpmsolver++", True)]
CASES = ([(mt, "multistep", 2, al, th, phi) for mt in ("noise", "x_start", "v", "score") for al, th in ALGOS
          for phi in (0., PHI)] +
         [("noise", m, o, al, th, phi) for m, o in FIXED if (m, o) != ("multistep", 2) for al, th in ALGOS
          for phi in (0., PHI)])


@pytest.mark.parametrize("model_type,method,order,algo,thr,phi", CASES)
def test_rows_match_reference_run_per_scale(guided_backend, model_type, method, order, algo, thr, phi):
    x = seeded(SHAPE, 11)
    d2z = model_type in ("noise", "v")
    kw = dict(steps=6, order=order, method=method, skip_type="time_uniform", denoise_to_zero=d2z,
              return_intermediate=True)
    yp, ip = product(model_type, algo, thr, phi=phi).sample(x.clone(), **kw)
    for rows, (yr, ir) in reference_rows(model_type, algo, thr, phi, lambda s, xr: s.sample(xr, **kw), x):
        np.testing.assert_array_equal(yp[rows].numpy(), yr.numpy())
        assert len(ip) == len(ir)
        for a, b in zip(ip, ir):
            np.testing.assert_array_equal(a[rows].numpy(), b.numpy())
    assert any(e[0] == "guided" for e in guided_backend.log)


@pytest.mark.parametrize("phi", [0., PHI])
def test_inverse_and_lower_order_final(guided_backend, phi):
    x = seeded(SHAPE, 12)
    for call in (lambda s, xr: s.inverse(xr, steps=5, order=2, method="multistep"),
                 lambda s, xr: s.sample(xr, steps=5, order=3, method="multistep", lower_order_final=False)):
        yp = call(product("noise", "dpmsolver++", False, phi=phi), x.clone())
        for rows, yr in reference_rows("noise", "dpmsolver++", False, phi, call, x):
            np.testing.assert_array_equal(yp[rows].numpy(), yr.numpy())


def rowwise_net(scales, phi):
    """What a user would pass to the reference for the adaptive solver: the per-row combine in eager fp32 torch."""
    s = torch.tensor(scales, dtype=torch.float32).reshape(-1, 1, 1, 1)
    inner, uc, c = inner_net(), torch.zeros(len(scales), 1), torch.ones(len(scales), 1)

    def net(x, t_input):
        out_u, out_c = inner(torch.cat([x] * 2), torch.cat([t_input] * 2), torch.cat([uc, c])).chunk(2)
        g = out_u + s * (out_c - out_u)
        if phi:
            r = torch.from_numpy(ratio64(out_c.numpy(), g.numpy())).reshape(-1, 1, 1, 1)
            g = phi * (g * r) + (1.0 - phi) * g
        return torch.where(s == 1, out_c, g)
    return net


def _adaptive(solver, x, order):
    with mock.patch("builtins.print") as pr:
        y = solver.sample(x.clone(), order=order, method="adaptive", atol=0.05, rtol=0.1)
        return y, pr.call_args[0][-1]


# (a v network without the rescale is left out: the reference would combine before the parameterisation, the product
# after it, as the reference's own CFG does)
@pytest.mark.parametrize("model_type,phi", [("noise", 0.), ("noise", PHI), ("v", PHI)])
@pytest.mark.parametrize("algo,thr", ALGOS)
def test_adaptive_matches_reference_with_rowwise_net(guided_backend, model_type, algo, thr, phi):
    ref, rns, _ = schedules("sd")
    x = seeded(SHAPE, 11)
    rs = ref.DPM_Solver(ref.model_wrapper(rowwise_net(SCALES, phi), rns, model_type=model_type), rns,
                        **_kw(algo, thr))
    yr, nfe_r = _adaptive(rs, x, 2)
    yp, nfe_p = _adaptive(product(model_type, algo, thr, phi=phi), x, 2)
    assert nfe_p == nfe_r
    err = np.abs(yp.numpy().astype(np.float64) - yr.numpy()).max() / max(np.abs(yr.numpy()).max(), 1e-30)
    assert err <= 1e-5


@pytest.mark.parametrize("algo,thr", ALGOS)
@pytest.mark.parametrize("phi", [0., PHI])
@pytest.mark.parametrize("method", ["multistep", "singlestep", "adaptive"])
def test_all_equal_scales_give_the_scalar_run(guided_backend, algo, thr, phi, method):
    x = seeded(SHAPE, 13)
    kw = dict(order=3, method=method)
    kw.update(dict(atol=0.05, rtol=0.1) if method == "adaptive" else dict(steps=6))
    with mock.patch("builtins.print"):
        y_vec = product("v", algo, thr, scales=torch.full((B,), 7.5), phi=phi).sample(x.clone(), **kw)
        y_one = product("v", algo, thr, scales=7.5, phi=phi).sample(x.clone(), **kw)
    np.testing.assert_array_equal(y_vec.numpy(), y_one.numpy())


@pytest.mark.parametrize("scale", [7.5, torch.tensor(7.5), torch.tensor([7.5]), [7.5]])
def test_scalar_forms_keep_the_one_scale_path(guided_backend, scale):
    x = seeded(SHAPE, 14)
    guided_backend.log.clear()
    y = product("noise", "dpmsolver++", True, scales=scale).sample(x.clone(), steps=5, order=2)
    log = list(guided_backend.log)
    guided_backend.log.clear()
    y_ref = product("noise", "dpmsolver++", True, scales=7.5).sample(x.clone(), steps=5, order=2)
    assert log == guided_backend.log and not any(e[0] == "guided" for e in log)
    np.testing.assert_array_equal(y.numpy(), y_ref.numpy())


def _log(be, scales, phi, thr):
    """(launches, log) of one sample() run."""
    be.log.clear()
    n0 = be.launches
    product("noise", "dpmsolver++", thr, scales=scales, phi=phi).sample(seeded(SHAPE, 5), steps=5, order=2)
    return be.launches - n0, list(be.log)


@pytest.mark.parametrize("thr", [False, True])
@pytest.mark.parametrize("phi", [0., PHI])
def test_launch_budget(guided_backend, thr, phi):
    """+0 launches per evaluation without thresholding, +1 with it (the guided noise materialised once), +2 with the
    rescale (the ratio pass; with thresholding the rescale already materialises its output)."""
    (n_vec, vec), (n_one, _) = _log(guided_backend, SCALES, phi, thr), _log(guided_backend, 7.5, phi, thr)
    n_plain, _ = _log(guided_backend, 7.5, 0., thr)
    nfe = 5
    assert n_vec - n_plain == (2 * nfe if phi else 0) + (nfe if thr else 0)
    assert n_vec - n_one == (nfe if thr and not phi else 0)
    assert vec.count(("ratio", 2)) == (nfe if phi else 0)
    assert sum(e[0] == "guided" for e in vec) == nfe        # every evaluation takes exactly one guided launch
    if thr:
        assert vec.count(("guided", 0)) == nfe              # FORM_NONE: the materialisation


def test_direct_model_fn_call(guided_backend):
    """WrappedModel.__call__, one time label for the batch and one per sample: row b is that of the one-scale call."""
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    x = seeded(SHAPE, 3)
    for model_type in ("noise", "x_start", "v", "score"):
        for phi in (0., PHI):
            mk = lambda s, n: new.model_wrapper(inner_net(), pns, model_type=model_type,
                                                guidance_type="classifier-free", condition=torch.ones(n, 1),
                                                unconditional_condition=torch.zeros(n, 1), guidance_scale=s,
                                                guidance_rescale=phi)
            for t in (torch.full((B,), 0.6), torch.linspace(0.9, 0.2, B)):
                got = mk(SCALES, B)(x, t).numpy()
                for b, s in enumerate(SCALES):
                    want = mk(s, 1)(x[b:b + 1], t[b:b + 1]).numpy()
                    np.testing.assert_array_equal(got[b:b + 1], want)


def test_invalid_scales_raise_before_the_network_runs(guided_backend):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    calls = []
    net = inner_net(calls)
    cfg = dict(guidance_type="classifier-free", condition=torch.ones(B, 1), unconditional_condition=torch.zeros(B, 1))
    for bad in (SCALES[:-1], torch.tensor(SCALES + [2.0])):
        fn = new.model_wrapper(net, pns, guidance_scale=bad, **cfg)
        with pytest.raises(ValueError):
            new.DPM_Solver(fn, pns).sample(seeded(SHAPE, 5), steps=3, order=2)
        with pytest.raises(ValueError):
            fn(seeded(SHAPE, 5), torch.full((B,), 0.5))
    assert calls == []
    with pytest.raises(ValueError):
        new.model_wrapper(net, pns, guidance_scale=torch.ones(2, 3), **cfg)
    with pytest.raises(ValueError):
        new.model_wrapper(net, pns, guidance_type="classifier", classifier_fn=lambda *a: a[0].sum(),
                          guidance_scale=torch.tensor(SCALES))
    fn = new.model_wrapper(net, pns, guidance_scale=torch.tensor(SCALES), **cfg)
    with pytest.raises(ValueError):
        new.DPM_Solver(fn, pns, algorithm_type="dpmsolver", reference_rounding=True)
    assert calls == []


def test_tensor_scale_outside_cfg_is_ignored_as_before(guided_backend):
    """An unconditional wrapper ignores guidance_scale: a tensor there changes nothing, reference_rounding included."""
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    fn = new.model_wrapper(lambda x, t: x * 0.5, pns, guidance_type="uncond", guidance_scale=torch.tensor(SCALES))
    assert not fn.per_sample_guidance and not fn.uses_cfg
    new.DPM_Solver(fn, pns, algorithm_type="dpmsolver", reference_rounding=True)


def test_nan_scale_gives_the_reference_row(guided_backend):
    scales = [7.5, float("nan"), 2.0]
    x = seeded((3, 2, 4, 4), 8)
    kw = dict(steps=4, order=2, method="multistep")
    yp = product("noise", "dpmsolver", False, scales=scales, batch=3).sample(x.clone(), **kw)
    ref, rns, _ = schedules("sd")
    fn = ref.model_wrapper(inner_net(), rns, guidance_type="classifier-free", condition=torch.ones(1, 1),
                           unconditional_condition=torch.zeros(1, 1), guidance_scale=float("nan"))
    yr = ref.DPM_Solver(fn, rns, algorithm_type="dpmsolver").sample(x[1:2].clone(), **kw)
    np.testing.assert_array_equal(yp[1:2].numpy(), yr.numpy())


def test_scales_are_converted_once_per_version(guided_backend):
    import dpm_solver_b200 as new
    _, _, pns = schedules("sd")
    s = torch.tensor(SCALES, dtype=torch.float64)
    fn = new.model_wrapper(inner_net(), pns, guidance_type="classifier-free", condition=torch.ones(B, 1),
                           unconditional_condition=torch.zeros(B, 1), guidance_scale=s)
    x = seeded(SHAPE, 1)
    a = fn._scales(x)
    assert a.dtype == torch.float32 and fn._scales(x) is a
    s[0] = 3.0                                    # an in-place write bumps the version: converted again
    b = fn._scales(x)
    assert b is not a and float(b[0]) == 3.0
    s32 = torch.tensor(SCALES)
    fn32 = new.model_wrapper(inner_net(), pns, guidance_type="classifier-free", condition=torch.ones(B, 1),
                             unconditional_condition=torch.zeros(B, 1), guidance_scale=s32)
    assert fn32._scales(x) is s32                 # already in the kernels' form: read in place


def _worker(rank, world, port, outdir):
    import sys
    for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    from dpm_solver_b200.distributed import shard_batch
    from helpers import product_schedule
    ops.set_backend(GuidedOracle())
    ns = product_schedule("sd")
    x = shard_batch(seeded((6, 2, 4, 4), 5)).contiguous()
    b = x.shape[0]
    fn = new.model_wrapper(inner_net(), ns, guidance_type="classifier-free", condition=torch.ones(b, 1),
                           unconditional_condition=torch.zeros(b, 1), guidance_scale=shard_batch(torch.tensor(SCALES)),
                           guidance_rescale=PHI)
    y = new.DPM_Solver(fn, ns, plan_broadcast=True, correcting_x0_fn="dynamic_thresholding").sample(
        x, steps=6, order=3, method="singlestep")
    np.save(os.path.join(outdir, f"y{rank}.npy"), y.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_shards_equal_single_process(tmp_path, guided_backend):
    import socket
    import dpm_solver_b200 as new
    from helpers import product_schedule
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    ns = product_schedule("sd")
    fn = new.model_wrapper(inner_net(), ns, guidance_type="classifier-free", condition=torch.ones(6, 1),
                           unconditional_condition=torch.zeros(6, 1), guidance_scale=SCALES, guidance_rescale=PHI)
    full = new.DPM_Solver(fn, ns, correcting_x0_fn="dynamic_thresholding").sample(
        seeded((6, 2, 4, 4), 5), steps=6, order=3, method="singlestep").numpy()
    got = np.concatenate([np.load(tmp_path / "y0.npy"), np.load(tmp_path / "y1.npy")])
    np.testing.assert_array_equal(got, full)
