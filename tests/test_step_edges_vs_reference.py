"""The numpy executor at the step kernels' edges, against the UNMODIFIED reference (oracle/_ref).

tests/test_gpu_step_edges.py holds the CUDA kernels to the numpy executor on edge-valued operands; this file is what
makes the executor a valid oracle there. Every public update method, model_fn, noise_prediction_fn and
data_prediction_fn of the product (its host logic on OracleBackend) and of the reference run on edge-valued x, model
buffers and networks (tests/step_edges.py: NaN, +-inf, -0, subnormals, overflowing values, numerators at the
constant division's guard), for every model type, with and without CFG and dynamic thresholding, both algorithms
and both solver types, and with 16-bit network outputs under `reference_rounding=True`. NaN must sit in the same
places and every other element must be bit-identical."""
import random

import numpy as np
import pytest
import torch

from cases import make_betas
from step_edges import assert_bits_equal, scatter_edges
from test_random_configs_vs_reference import pytestmark, reference_module  # noqa: F401  (same skip rule)

SHAPE = (2, 3, 8, 8)


def edge_tensor(shape, seed, dtype=torch.float32, scale=1.0):
    rng = np.random.default_rng(seed)
    v = (rng.standard_normal(int(np.prod(shape))) * scale).astype(np.float32)
    scatter_edges({"v": v}, {"v": dtype}, rng, frac=0.5)
    return torch.from_numpy(v).reshape(shape).to(dtype)


def edge_net(seed, dtype):
    """A network whose k-th call returns the k-th edge-valued tensor (plus a condition term under CFG)."""
    calls = [0]

    def net(x, t, *cond):
        calls[0] += 1
        o = edge_tensor(x.shape, seed * 1000 + calls[0], torch.float32, 1.3)
        if cond:
            o = o + 0.05 * cond[0].reshape(-1, 1, 1, 1)
        return o.to(dtype)
    return net


def run(mod, c):
    _, betas = make_betas(c["schedule"])
    ns = mod.NoiseScheduleVP("discrete", betas=torch.from_numpy(betas))
    net = edge_net(c["seed"], c["net_dtype"])
    B = SHAPE[0]
    if c["cfg"] is not None:
        fn = mod.model_wrapper(net, ns, model_type=c["model_type"], guidance_type="classifier-free",
                               condition=torch.ones(B, 1), unconditional_condition=torch.zeros(B, 1),
                               guidance_scale=c["cfg"])
    else:
        fn = mod.model_wrapper(net, ns, model_type=c["model_type"])
    kw = dict(reference_rounding=True) if c["rr"] and mod is not reference_module() else {}
    s = mod.DPM_Solver(fn, ns, algorithm_type=c["algo"],
                       correcting_x0_fn="dynamic_thresholding" if c["thr"] else None, **kw)
    x = edge_tensor(SHAPE, c["seed"])
    t = lambda v: torch.tensor(v)
    ts = sorted(c["ts"], reverse=True)
    ms = [edge_tensor(SHAPE, c["seed"] + 7 + i) for i in range(3)]
    tp = [t(ts[0]), t(ts[1]), t(ts[2])]
    k, st = c["kind"], c["st"]

    def flat(o):
        if isinstance(o, tuple):
            return [o[0]] + [o[1][key] for key in sorted(o[1])]
        return [o]
    if k == "first":
        return flat(s.dpm_solver_first_update(x, t(ts[0]), t(ts[1]), return_intermediate=True))
    if k == "ss2":
        return flat(s.singlestep_dpm_solver_second_update(x, t(ts[0]), t(ts[1]), r1=0.5, return_intermediate=True,
                                                          solver_type=st))
    if k == "ss3":
        return flat(s.singlestep_dpm_solver_third_update(x, t(ts[0]), t(ts[1]), return_intermediate=True,
                                                         solver_type=st))
    if k == "ssu":
        return flat(s.singlestep_dpm_solver_update(x, t(ts[0]), t(ts[1]), c["order"], return_intermediate=True,
                                                   solver_type=st))
    if k == "ms2":
        return flat(s.multistep_dpm_solver_second_update(x, ms[1:], tp[1:], t(ts[3]), solver_type=st))
    if k == "ms3":
        return flat(s.multistep_dpm_solver_third_update(x, ms, tp, t(ts[3]), solver_type=st))
    if k == "msu":
        o = c["order"]
        return flat(s.multistep_dpm_solver_update(x, ms[3 - o:], tp[3 - o:], t(ts[3]), o, solver_type=st))
    return [s.model_fn(x, t(ts[0])), s.noise_prediction_fn(x, t(ts[0])), s.data_prediction_fn(x, t(ts[0]))]


KINDS = ["first", "ss2", "ss3", "ssu", "ms2", "ms3", "msu", "fns"]


@pytest.mark.parametrize("kind", KINDS)
def test_executor_matches_reference_at_edges(oracle_backend, kind):
    import dpm_solver_b200 as new
    ref = reference_module()
    compared = 0
    for i in range(24):
        rng = random.Random(7000 + 100 * KINDS.index(kind) + i)
        rr = i % 4 == 3
        c = dict(schedule=rng.choice(["sd", "ddpm_linear", "iddpm_cosine"]), kind=kind, seed=rng.randint(0, 10 ** 6),
                 algo=rng.choice(["dpmsolver++", "dpmsolver"]), st=rng.choice(["dpmsolver", "taylor"]),
                 model_type="noise" if rr else ["noise", "x_start", "v", "score"][i % 4],
                 cfg=rng.choice([None, 1.0, 3.5, 7.5]), order=rng.choice([1, 2, 3]),
                 ts=[rng.uniform(0.002, 1.0) for _ in range(4)], rr=rr,
                 net_dtype=rng.choice([torch.bfloat16, torch.float16]) if rr else torch.float32)
        c["thr"] = c["algo"] == "dpmsolver++" and i % 3 != 0
        try:
            a = run(ref, c)
        except Exception as e:   # what the reference rejects must be rejected the same way
            with pytest.raises(type(e)):
                run(new, c)
            continue
        b = run(new, c)
        assert len(a) == len(b), c
        for j, (u, v) in enumerate(zip(a, b)):
            if rr and (kind == "fns" or j > 0) and u.dtype != torch.float32:
                # raw 16-bit network outputs (model_fn, the intermediates dict): the product hands them on widened to
                # fp32 (exactly), the reference in the network's type
                u, v = u.float(), v.float()
            assert u.dtype == v.dtype and u.shape == v.shape, (c, j)
            assert_bits_equal(v, u, "output %d of %s" % (j, c))
            compared += 1
    assert compared >= 24
