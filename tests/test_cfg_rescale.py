"""Guidance rescale (`model_wrapper(..., guidance_rescale=phi)`) on the CPU: the product's host logic, driven by a
numpy executor that computes the per-sample ratio in fp64 and the rescale in fp32, against the UNMODIFIED reference
fed a network that does the CFG combine and the rescale itself in eager fp32 torch."""
import dataclasses
import os
from unittest import mock

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from cases import exact_net, make_betas, seeded
from oracle_backend import OracleBackend, _np

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S, PHI, B, SHAPE = 3.5, 0.7, 3, (3, 2, 4, 4)


def ratio64(c, g):
    """fl32(std(c_b)) / fl32(std(g_b)) per sample: unbiased, fp64, each std rounded to fp32 once, fp32 division."""
    with np.errstate(all="ignore"):
        c64 = c.reshape(c.shape[0], -1).astype(np.float64)
        g64 = g.reshape(g.shape[0], -1).astype(np.float64)
        return (np.std(c64, axis=1, ddof=1).astype(f32) / np.std(g64, axis=1, ddof=1).astype(f32)).astype(f32)


class RescaleOracle(OracleBackend):
    """OracleBackend plus the rescale: r in fp64 numpy, g' = phi*(g*r) + psi*g in fp32 numpy."""

    def cfg_rescale_ratio(self, e_cond, e_uncond, guidance):
        self.launches += 2
        self.log.append(("ratio", 2))
        c, u = _np(e_cond), _np(e_uncond)
        g = (u + f32(guidance) * (c - u)).astype(f32)
        return torch.from_numpy(ratio64(c, g))

    def _model_value(self, a, thr=None):
        if a.ratio is None:
            return super()._model_value(a, thr)
        c, u = _np(a.e_cond), _np(a.e_uncond)
        with np.errstate(all="ignore"):
            g = (u + f32(a.guidance) * (c - u)).astype(f32)
            r = np.repeat(_np(a.ratio), a.per_sample).reshape(g.shape)
            gp = (f32(a.phi) * (g * r) + f32(1.0 - a.phi) * g).astype(f32)
        return super()._model_value(dataclasses.replace(a, n_model=1, e_cond=torch.from_numpy(gp), e_uncond=None,
                                                        ratio=None), thr)


@pytest.fixture()
def rescale_backend():
    from dpm_solver_b200 import ops
    be = RescaleOracle()
    old = ops._backend
    ops.set_backend(be)
    yield be
    ops.set_backend(old)


def inner_net(calls=None):
    """The network of both runs: the conditional half differs from the unconditional one in scale and offset, so
    std(out_c) != std(g). `calls` records (first time label, input shape) per call."""
    def net(x, t, c):
        if calls is not None:
            calls.append((float(t.reshape(-1)[0]), tuple(x.shape)))
        return exact_net(x.float(), t) * (1. + 0.3 * c.reshape(-1, 1, 1, 1)) + 0.05 * c.reshape(-1, 1, 1, 1)
    return net


def ref_rescaled_net(inner, uc, c, s, phi):
    """What a user would pass to the reference: the CFG combine and the rescale in eager fp32 torch."""
    def net(x, t_input):
        out = inner(torch.cat([x] * 2), torch.cat([t_input] * 2), torch.cat([uc, c]))
        out_u, out_c = out.chunk(2)
        g = out_u + s * (out_c - out_u)
        r = torch.from_numpy(ratio64(out_c.numpy(), g.numpy())).reshape(-1, *([1] * (g.dim() - 1)))
        return phi * (g * r) + (1.0 - phi) * g
    return net


def schedules(sched):
    from oracle import ref_loader
    from helpers import product_schedule
    ref = ref_loader.load("dpm_solver_pytorch")
    kind, betas = make_betas(sched)
    rns = ref.NoiseScheduleVP("discrete", betas=torch.from_numpy(betas)) if kind == "discrete" else \
        ref.NoiseScheduleVP("linear", continuous_beta_0=0.1, continuous_beta_1=20.)
    return ref, rns, product_schedule(sched)


def make_pair(model_type, algo, thresholding, phi=PHI, s=S, sched="sd"):
    """(reference solver, product solver, reference calls, product calls)."""
    import dpm_solver_b200 as new
    ref, rns, pns = schedules(sched)
    uc, c = torch.zeros(B, 1), torch.ones(B, 1)
    rc, pc = [], []
    rfn = ref.model_wrapper(ref_rescaled_net(inner_net(rc), uc, c, s, phi), rns, model_type=model_type)
    pfn = new.model_wrapper(inner_net(pc), pns, model_type=model_type, guidance_type="classifier-free",
                            condition=c, unconditional_condition=uc, guidance_scale=s, guidance_rescale=phi)
    kw = dict(algorithm_type=algo, correcting_x0_fn="dynamic_thresholding" if thresholding else None)
    return ref.DPM_Solver(rfn, rns, **kw), new.DPM_Solver(pfn, pns, **kw), rc, pc


METHODS = [("multistep", 1), ("multistep", 2), ("multistep", 3), ("singlestep", 2), ("singlestep", 3),
           ("singlestep_fixed", 2), ("adaptive", 2), ("adaptive", 3)]
ALGOS = [("dpmsolver", False), ("dpmsolver", True), ("dpmsolver++", False), ("dpmsolver++", True)]


@pytest.mark.parametrize("model_type", ["noise", "x_start", "v", "score"])
@pytest.mark.parametrize("method,order", METHODS)
@pytest.mark.parametrize("algo,thr", ALGOS)
def test_sample_matches_reference_with_eager_rescale(rescale_backend, model_type, method, order, algo, thr):
    rs, ps, rc, pc = make_pair(model_type, algo, thr)
    x = seeded(SHAPE, 11)
    if method == "adaptive":
        kw = dict(order=order, method=method, atol=0.05, rtol=0.1)
        with mock.patch("builtins.print") as pr:
            yr = rs.sample(x.clone(), **kw)
            nfe_r = pr.call_args[0][-1]
        with mock.patch("builtins.print") as pr:
            yp = ps.sample(x.clone(), **kw)
            nfe_p = pr.call_args[0][-1]
        # the error estimate is a mean whose summation order differs from torch's (DESIGN.md section 2)
        assert nfe_p == nfe_r
        err = np.abs(yp.numpy().astype(np.float64) - yr.numpy()).max() / max(np.abs(yr.numpy()).max(), 1e-30)
        assert err <= 1e-5
        return
    d2z = model_type in ("noise", "v")
    kw = dict(steps=6, order=order, method=method, skip_type="time_uniform", denoise_to_zero=d2z,
              return_intermediate=True)
    yr, ir = rs.sample(x.clone(), **kw)
    yp, ip = ps.sample(x.clone(), **kw)
    assert pc == rc                                  # the same network calls, in the same order
    assert len(ip) == len(ir)
    for a, b in zip(ip, ir):
        np.testing.assert_array_equal(a.numpy(), b.numpy())
    np.testing.assert_array_equal(yp.numpy(), yr.numpy())
    assert ("ratio", 2) in rescale_backend.log


@pytest.mark.parametrize("model_type", ["noise", "x_start", "v", "score"])
def test_model_fn_direct_call(rescale_backend, model_type):
    """WrappedModel.__call__, one time label for the batch and one per sample."""
    rs, ps, rc, pc = make_pair(model_type, "dpmsolver", False)
    x = seeded(SHAPE, 3)
    for t in (torch.full((B,), 0.6), torch.tensor([0.9, 0.5, 0.2])):
        np.testing.assert_array_equal(ps._wrapped(x, t).numpy(), rs.model(x, t).numpy())


def _log(be, phi, s=S, uncond=True):
    import dpm_solver_b200 as new
    from helpers import product_schedule
    ns = product_schedule("sd")
    be.log.clear()
    kw = dict(guidance_type="classifier-free", condition=torch.ones(B, 1), guidance_scale=s,
              unconditional_condition=torch.zeros(B, 1) if uncond else None)
    if phi is not None:
        kw["guidance_rescale"] = phi
    fn = new.model_wrapper(inner_net([]), ns, **kw)
    y = new.DPM_Solver(fn, ns).sample(seeded(SHAPE, 5), steps=5, order=2)
    return list(be.log), y


def test_phi_zero_is_plain_cfg(rescale_backend):
    log_none, y_none = _log(rescale_backend, None)
    log_zero, y_zero = _log(rescale_backend, 0.0)
    assert log_zero == log_none and ("ratio", 2) not in log_none
    np.testing.assert_array_equal(y_zero.numpy(), y_none.numpy())
    log_on, _ = _log(rescale_backend, PHI)
    assert log_on.count(("ratio", 2)) == 5          # one ratio pass per CFG evaluation


@pytest.mark.parametrize("s,uncond", [(1.0, True), (S, False)])
def test_bypassed_cfg_launches_nothing_extra(rescale_backend, s, uncond):
    log_off, y_off = _log(rescale_backend, 0.0, s, uncond)
    log_on, y_on = _log(rescale_backend, PHI, s, uncond)
    assert log_on == log_off
    np.testing.assert_array_equal(y_on.numpy(), y_off.numpy())


def test_invalid_combinations_raise():
    import dpm_solver_b200 as new
    from helpers import product_schedule
    ns = product_schedule("sd")
    net = inner_net([])
    for gt in ("uncond", "classifier"):
        with pytest.raises(ValueError):
            new.model_wrapper(net, ns, guidance_type=gt, guidance_rescale=0.5)
    for bad in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError):
            new.model_wrapper(net, ns, guidance_type="classifier-free", guidance_rescale=bad)
    fn = new.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B, 1),
                           unconditional_condition=torch.zeros(B, 1), guidance_scale=S, guidance_rescale=PHI)
    with pytest.raises(ValueError):
        new.DPM_Solver(fn, ns, algorithm_type="dpmsolver", reference_rounding=True)
    new.model_wrapper(net, ns, guidance_type="uncond", guidance_rescale=0.0)     # phi = 0 is accepted everywhere


def test_executor_without_ratio_pass_raises(oracle_backend):
    import dpm_solver_b200 as new
    from helpers import product_schedule
    ns = product_schedule("sd")
    fn = new.model_wrapper(inner_net([]), ns, guidance_type="classifier-free", condition=torch.ones(B, 1),
                           unconditional_condition=torch.zeros(B, 1), guidance_scale=S, guidance_rescale=PHI)
    with pytest.raises(RuntimeError, match="cfg_rescale_ratio"):
        new.DPM_Solver(fn, ns).sample(seeded(SHAPE, 5), steps=3, order=2)


def _worker(rank, world, port, outdir):
    import sys
    for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import dpm_solver_b200 as new
    from dpm_solver_b200 import ops
    from dpm_solver_b200.distributed import shard_bounds, shard_batch
    from helpers import product_schedule
    ops.set_backend(RescaleOracle())
    ns = product_schedule("sd")
    lo, hi = shard_bounds(6, rank, world)
    fn = new.model_wrapper(inner_net([]), ns, guidance_type="classifier-free", condition=torch.ones(hi - lo, 1),
                           unconditional_condition=torch.zeros(hi - lo, 1), guidance_scale=S, guidance_rescale=PHI)
    x = seeded((6, 2, 4, 4), 5)
    y = new.DPM_Solver(fn, ns, plan_broadcast=True).sample(shard_batch(x).contiguous(), steps=6, order=3,
                                                           method="singlestep")
    np.save(os.path.join(outdir, f"y{rank}.npy"), y.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_shards_equal_single_process(tmp_path, rescale_backend):
    import socket
    import dpm_solver_b200 as new
    from helpers import product_schedule
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    ns = product_schedule("sd")
    fn = new.model_wrapper(inner_net([]), ns, guidance_type="classifier-free", condition=torch.ones(6, 1),
                           unconditional_condition=torch.zeros(6, 1), guidance_scale=S, guidance_rescale=PHI)
    full = new.DPM_Solver(fn, ns).sample(seeded((6, 2, 4, 4), 5), steps=6, order=3, method="singlestep").numpy()
    got = np.concatenate([np.load(tmp_path / "y0.npy"), np.load(tmp_path / "y1.npy")])
    np.testing.assert_array_equal(got, full)
