"""The multi-condition executor (MultiOracle) at the step kernels' edges, against the UNMODIFIED reference composition.

tests/test_gpu_cfg_multi_edges.py holds dpm_step_multi to MultiOracle on edge-valued operands; this file is what makes
MultiOracle a valid oracle there. The product's host logic on MultiOracle and the reference composed the way a user
would compose it (the reference's model_wrapper per condition at guidance_scale=1, combined left to right in eager
fp32 torch, as test_cfg_multi.reference_composed does) run the first, second and third-order updates and the model
functions on edge-valued x, model buffers and networks (tests/step_edges.py), with K = 2, 3 and 4 conditions, every
model type, both algorithms, with and without dynamic thresholding, and scales that include 0, -0, negative values,
NaN and infinities. NaN must sit in the same places and every other element must be bit-identical. A zero scale
keeps its condition in the combine (0 * inf is NaN), and a NaN or infinite scale reaches every element."""
import random

import pytest
import torch

from step_edges import assert_bits_equal
from test_cfg_multi import multi_backend  # noqa: F401  (fixture)
from test_cfg_rescale import schedules
from test_random_configs_vs_reference import pytestmark  # noqa: F401  (same skip rule)
from test_step_edges_vs_reference import edge_tensor

SHAPE = (2, 3, 8, 8)
B = SHAPE[0]
FINITE_SCALES = [0.0, -0.0, 1.0, -1.5, 3.5, 7.5]
SPECIAL_SCALES = [0.0, -0.0, float("nan"), float("inf"), float("-inf")]


def edge_net(seed):
    """A network whose output for one block of B rows is an edge-valued tensor determined by the evaluation time and
    the block's condition value alone, so that one call on the K+1 stacked blocks (the product) and K+1 calls on one
    block each (the reference composition) see the same outputs."""
    def net(x, t, c):
        tk = int(round(float(t.reshape(-1)[0]) * 1000))
        v = c[:, 0]
        out = torch.empty(x.shape, dtype=torch.float32)
        for val in sorted(set(v.tolist())):
            rows = (v == val).nonzero().reshape(-1)
            s = (seed * 7919 + tk * 131 + int(val) * 17) % (2 ** 31)
            out[rows] = edge_tensor((len(rows),) + tuple(x.shape[1:]), s, torch.float32, 1.3)
        return out
    return net


def conds(K):
    return [torch.full((B, 1), float(k + 1)) for k in range(K)]


def product_fn(pns, c):
    import dpm_solver_b200 as new
    return new.model_wrapper(edge_net(c["seed"]), pns, model_type=c["model_type"], guidance_type="classifier-free",
                             condition=conds(c["K"]), unconditional_condition=torch.zeros(B, 1),
                             guidance_scale=c["scales"])


def reference_fn(ref, rns, c):
    uc = torch.zeros(B, 1)
    fs = [ref.model_wrapper(edge_net(c["seed"]), rns, model_type=c["model_type"], guidance_type="classifier-free",
                            condition=cc, unconditional_condition=uc, guidance_scale=1.0) for cc in [uc] + conds(c["K"])]

    def composed(x, t):
        eu = fs[0](x, t)
        e = eu
        for s, f in zip(c["scales"], fs[1:]):
            e = e + s * (f(x, t) - eu)
        return e
    return composed


def run(side, c):
    ref, rns, pns = schedules("sd")
    if side == "reference":
        s = ref.DPM_Solver(reference_fn(ref, rns, c), rns, algorithm_type=c["algo"],
                           correcting_x0_fn="dynamic_thresholding" if c["thr"] else None)
    else:
        import dpm_solver_b200 as new
        s = new.DPM_Solver(product_fn(pns, c), pns, algorithm_type=c["algo"],
                           correcting_x0_fn="dynamic_thresholding" if c["thr"] else None)
    x = edge_tensor(SHAPE, c["seed"])
    t = lambda v: torch.tensor(v)
    ts = sorted(c["ts"], reverse=True)
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
    if k in ("ms2", "ms3"):
        # the multistep updates only combine buffers: sample() runs them on the network's outputs, evaluated inside
        # the fused step of the previous update
        o = s.sample(x, steps=4, order=int(k[2]), method="multistep", skip_type="time_uniform", t_start=ts[0],
                     t_end=ts[3], solver_type=st, return_intermediate=True)
        return [o[0]] + list(o[1])
    return [s.model_fn(x, t(ts[0])), s.noise_prediction_fn(x, t(ts[0])), s.data_prediction_fn(x, t(ts[0]))]


KINDS = ["first", "ss2", "ss3", "ms2", "ms3", "fns"]
MODELS = ["noise", "x_start", "v", "score"]


@pytest.mark.parametrize("K", [2, 3, 4])
@pytest.mark.parametrize("kind", KINDS)
def test_multi_executor_matches_reference_composition_at_edges(multi_backend, kind, K):  # noqa: F811
    compared, specials = 0, set()
    for i in range(8):
        rng = random.Random(31000 + 1000 * K + 100 * KINDS.index(kind) + i)
        algo = ["dpmsolver++", "dpmsolver"][i % 2]
        # one scale of each case at 0 or -0 (half of the cases) or NaN or +-inf (the other half, all outputs non-finite)
        scales = [rng.choice(FINITE_SCALES) for _ in range(K)]
        scales[i % K] = SPECIAL_SCALES[i % 2] if i < 4 else SPECIAL_SCALES[2 + i % 3]
        c = dict(kind=kind, K=K, seed=rng.randint(0, 10 ** 6), algo=algo, model_type=MODELS[(i // 2) % 4],
                 st=rng.choice(["dpmsolver", "taylor"]), ts=[rng.uniform(0.002, 1.0) for _ in range(4)],
                 thr=algo == "dpmsolver++" and i % 4 != 0, scales=scales)
        specials.update(repr(v) for v in scales)
        a = run("reference", c)
        b = run("product", c)
        assert len(a) == len(b), c
        for j, (u, v) in enumerate(zip(a, b)):
            assert u.dtype == v.dtype and u.shape == v.shape, (c, j)
            assert_bits_equal(v, u, "output %d of %s" % (j, c))
            compared += 1
    assert any(e[0] == "multi" for e in multi_backend.log)
    assert {"0.0", "-0.0", "nan"} <= specials and ({"inf", "-inf"} & specials), specials
    assert compared >= 8
