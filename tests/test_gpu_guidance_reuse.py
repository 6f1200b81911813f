"""One long-lived solver per guidance feature (CFG-Zero*, CFG++, regional masks) on the H100, under the invariant of
tests/test_gpu_solver_reuse.py: every call returns the bits a fresh wrapper and solver return for that call. Between
calls the tests edit converted masks and per-sample scale tensors in place, switch x between row-major and
channels_last and between two shapes of one size, change cfg_zero_init_steps and cfg_pp on the wrapper, alternate
sample() and inverse() with other steps, orders and t_end, and stop runs with an exception raised by user code."""
import pytest
import torch

from gpu_configs import same_bits
from test_cfg_pp import product_schedule

pytestmark = pytest.mark.gpu
B = 3
S1, S2 = (B, 4, 16, 16), (B, 8, 8, 16)          # one size per sample, other shapes: a [.., 16] mask fits both


class Boom(RuntimeError):
    pass


def make_net(raise_at=None):
    """Products and sums only; raises Boom at its call number `raise_at[0]` (1-based) when set, counting in raise_at[1]."""
    def net(x, t, c):
        if raise_at is not None:
            raise_at[1] += 1
            if raise_at[1] == raise_at[0]:
                raise Boom("network call %d" % raise_at[1])
        cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
        tt = t.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
        return 0.45 * x + 0.05 * cc * x - 0.1 + 0.05 * cc + 1e-4 * tt
    return net


def xs(seed, shape=S1, cl=False, dtype=torch.float32):
    x = torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(dtype).cuda()
    return x.contiguous(memory_format=torch.channels_last) if cl else x


def wrapper(ns, mt, net=None, **kw):
    import dpm_solver_b200 as new
    kw.setdefault("condition", torch.ones(B, 1).cuda())
    return new.model_wrapper(net or make_net(), ns, model_type=mt, guidance_type="classifier-free",
                             unconditional_condition=torch.zeros(B, 1).cuda(), **kw)


def run(s, x, inverse=False, **skw):
    return (s.inverse if inverse else s.sample)(x, **skw)


# ---- regional masks ------------------------------------------------------------------------------------------------

def _masks():
    g = torch.Generator().manual_seed(4)
    q = lambda shape: torch.randint(-4, 9, shape, generator=g).float() * 0.25
    return [q((B, 1, 1, 16)).to(torch.bfloat16).cuda(),      # converted (bf16)
            q((16,)),                                        # converted (on the CPU)
            q((B, 1, 1, 1)).cuda()]                          # read in place


@pytest.mark.parametrize("thr", [False, True])
def test_masked_wrapper_across_layouts_shapes_and_edits(cuda_backend, thr):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    conds = [torch.full((B, 1), float(k + 1)).cuda() for k in range(3)]
    scales = [7.5, -2.0, 3.0]
    masks = _masks()
    kw = dict(algorithm_type="dpmsolver++", correcting_x0_fn="dynamic_thresholding" if thr else None)
    s = new.DPM_Solver(wrapper(ns, "noise", condition=conds, guidance_scale=scales, guidance_mask=masks), ns, **kw)
    skw = dict(steps=6, order=2)
    # (an edit is followed by a call of the previous call's shape and layout, so that only the version tells them apart)
    calls = [(1, S1, False, None), (1, S1, True, None), (2, S2, False, None),
             (1, S2, False, lambda: masks[0].mul_(-1)),      # bf16, converted: its copy must follow the edit
             (1, S1, True, None), (2, S1, True, lambda: masks[1].add_(0.5)),      # on the CPU, converted
             (2, S2, True, None), (3, S2, True, lambda: masks[2].mul_(2)), (3, S1, False, None), (2, S2, False, None)]
    for i, (seed, shape, cl, edit) in enumerate(calls):
        if edit is not None:
            edit()
        x = xs(seed, shape, cl)
        got = s.sample(x, **skw)
        fresh = new.DPM_Solver(wrapper(ns, "noise", condition=conds, guidance_scale=scales,
                                       guidance_mask=[m.clone() for m in masks]), ns, **kw)
        assert same_bits(got, fresh.sample(x.clone(), **skw)), (i, shape, cl)


# ---- CFG++ ---------------------------------------------------------------------------------------------------------

def test_cfgpp_solver_across_calls(cuda_backend):
    import dpm_solver_b200 as new
    ns = product_schedule("noise")
    w = torch.tensor([0.6, 1.0, 7.5]).cuda()
    fn = wrapper(ns, "noise", guidance_scale=w, cfg_pp=True)
    s = new.DPM_Solver(fn, ns, algorithm_type="dpmsolver++")
    calls = [(False, dict(steps=6, order=2), None), (True, dict(steps=5, order=1), None),
             (False, dict(steps=6, order=2), lambda: w.copy_(torch.tensor([0.2, 2.0, 1.0]))),
             (False, dict(steps=8, order=1, t_end=0.05), None), (True, dict(steps=6, order=2), None),
             (False, dict(steps=6, order=2, t_end=0.05), lambda: w.mul_(0.5)),
             (False, dict(steps=6, order=2), lambda: setattr(fn, "cfg_pp", False)),   # plain CFG on the same plans
             (False, dict(steps=6, order=2), lambda: setattr(fn, "cfg_pp", True)),
             # plain CFG first on new sampling arguments, then CFG++ on them: its plan must carry g
             (False, dict(steps=7, order=2), lambda: setattr(fn, "cfg_pp", False)),
             (False, dict(steps=7, order=1), None),
             (False, dict(steps=7, order=2), lambda: setattr(fn, "cfg_pp", True)),
             (False, dict(steps=7, order=1), None),
             (True, dict(steps=5, order=1), None)]
    for i, (inverse, skw, edit) in enumerate(calls):
        if edit is not None:
            edit()
        x = xs(10 + i % 3)
        got = run(s, x, inverse, **skw)
        ref = new.DPM_Solver(wrapper(ns, "noise", guidance_scale=w.clone(), cfg_pp=fn.cfg_pp), ns,
                             algorithm_type="dpmsolver++")
        assert same_bits(got, run(ref, x.clone(), inverse, **skw)), (i, inverse, skw)


# ---- CFG-Zero* -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("solver", ["dpm", "unipc"])
def test_cfgzero_solver_across_calls(cuda_backend, solver):
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    per_sample = solver == "dpm"               # (UniPC takes one scale)
    w = torch.tensor([4.5, 1.0, 2.5]).cuda() if per_sample else torch.tensor(4.5).cuda()
    fn = wrapper(ns, "flow", guidance_scale=w, cfg_zero_star=True, cfg_zero_init_steps=1)
    mk = (lambda f: new.UniPC(f, ns)) if solver == "unipc" else (lambda f: new.DPM_Solver(f, ns))
    s = mk(fn)
    edits = [None, lambda: w.mul_(-1.0).add_(2.0), lambda: setattr(fn, "cfg_zero_init_steps", 3),
             lambda: setattr(fn, "cfg_zero_init_steps", 0), lambda: w.fill_(1.0),
             lambda: setattr(fn, "cfg_zero_init_steps", 100)]
    for i, edit in enumerate(edits):
        if edit is not None:
            edit()
        for cl in (False, True):
            x = xs(20 + i, cl=cl)
            skw = dict(steps=6, order=2 if cl else 3)
            got = s.sample(x, **skw)
            ref = mk(wrapper(ns, "flow", guidance_scale=w.clone(), cfg_zero_star=True,
                             cfg_zero_init_steps=fn.cfg_zero_init_steps))
            assert same_bits(got, ref.sample(x.clone(), **skw)), (i, cl)


@pytest.mark.parametrize("cfz", [False, True])
@pytest.mark.parametrize("solver", ["dpm", "unipc"])
def test_one_scale_tensor_edited_to_one_and_back(cuda_backend, solver, cfz):
    """A one-element scale tensor set to 1 in place bypasses the halves (the network gets B rows, not 2B) and set back
    combines them again: the model-input time rows of the solver's cached tables must follow (they were cached for the
    first run's row count). Every run, denoise_to_zero included, is a fresh solver's."""
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    w = torch.tensor([4.5]).cuda()
    kw = dict(cfg_zero_star=True, cfg_zero_init_steps=1) if cfz else {}
    mk = (lambda f: new.UniPC(f, ns)) if solver == "unipc" else (lambda f: new.DPM_Solver(f, ns))
    s = mk(wrapper(ns, "flow", guidance_scale=w, **kw))
    for i, v in enumerate([4.5, 1.0, 3.0, 1.0, 1.0, 2.0]):
        w.fill_(v)
        x = xs(50 + i)
        skw = dict(steps=5, order=2, denoise_to_zero=i >= 4)
        got = s.sample(x, **skw)
        assert same_bits(got, mk(wrapper(ns, "flow", guidance_scale=w.clone(), **kw)).sample(x.clone(), **skw)), (i, v)


# ---- a run stopped by an exception ------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [1, 3])
def test_run_stopped_by_the_network(cuda_backend, k):
    """The network raises at its call k of a CFG-Zero* run on a bf16 x (fp32 state: the caller's tensor is what the
    network receives); the next runs and a direct data_prediction_fn call are a fresh solver's."""
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    plan = [None, 0]
    fn = wrapper(ns, "flow", net=make_net(plan), guidance_scale=4.5, cfg_zero_star=True, cfg_zero_init_steps=2)
    s = new.DPM_Solver(fn, ns)
    x, x2 = xs(30, dtype=torch.bfloat16), xs(31, dtype=torch.bfloat16)
    plan[:] = [k, 0]
    with pytest.raises(Boom):
        s.sample(x, steps=6, order=2)
    plan[:] = [None, 0]
    fresh = lambda: new.DPM_Solver(wrapper(ns, "flow", guidance_scale=4.5, cfg_zero_star=True, cfg_zero_init_steps=2),
                                   ns)
    t = torch.full((B,), 0.5, device="cuda")
    assert same_bits(s.data_prediction_fn(x2, t), fresh().data_prediction_fn(x2.clone(), t))
    assert same_bits(s.sample(x2, steps=6, order=2), fresh().sample(x2.clone(), steps=6, order=2))
    assert plan[1] == 1 + 6 - 2


@pytest.mark.parametrize("k", [0, 2])
def test_run_stopped_during_zero_init(cuda_backend, k):
    """A correcting_xt_fn raises at step k while zero-init evaluations are left: the count does not leak into a direct
    data_prediction_fn call (which must call the network) or into the next run."""
    import dpm_solver_b200 as new
    ns = product_schedule("flow")
    plan = [None, 0]
    stop = [k]

    def corr(x, t, step):
        if step == stop[0]:
            raise Boom("step %d" % step)
        return x
    fn = wrapper(ns, "flow", net=make_net(plan), guidance_scale=4.5, cfg_zero_star=True, cfg_zero_init_steps=5)
    s = new.DPM_Solver(fn, ns, correcting_xt_fn=corr)
    with pytest.raises(Boom):
        s.sample(xs(40), steps=6, order=2)
    stop[0] = -1
    x2 = xs(41)
    fresh = new.DPM_Solver(wrapper(ns, "flow", guidance_scale=4.5, cfg_zero_star=True, cfg_zero_init_steps=5), ns,
                           correcting_xt_fn=corr)
    t = torch.full((B,), 0.5, device="cuda")
    n0 = plan[1]
    assert same_bits(s.data_prediction_fn(x2, t), fresh.data_prediction_fn(x2.clone(), t))
    assert plan[1] == n0 + 1
    assert same_bits(s.sample(x2, steps=6, order=2), fresh.sample(x2.clone(), steps=6, order=2))
