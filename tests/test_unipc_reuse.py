"""One long-lived `UniPC` solver serving whatever arrives: other sampling arguments, `inverse()`, the variant changed as an
attribute, thresholding switched through `correcting_x0_fn`, more configurations than its caches hold, a schedule edited
in place, other shapes and layouts of one numel, and a `model_fn` shared with a long-lived DPM_Solver. UniPC keeps its
plans in DPM_Solver's per-instance plan and table caches under its own key. Invariant throughout: a call on the
long-lived solver returns exactly the bits a fresh solver returns for that call.

Each test runs on the numpy executor (CPU tensors) and on the device, so the host-side cache logic is exercised without
a GPU. On the device only: a steady-state call reads nothing back, and one `DiffEditCorrector` as UniPC's
`correcting_xt_fn` across runs equals the numpy executor driving the notebook's corrector_fn with the same normals."""
import contextlib
import random

import pytest
import torch

from cases import seeded
from flow_unipc_configs import FlowRig
from gpu_configs import backend, same_bits
from unipc_oracle import UniPCOracle

DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


@pytest.fixture(autouse=True)
def peak_memory():
    if not torch.cuda.is_available():
        yield
        return
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


@contextlib.contextmanager
def executor(dev):
    """The numpy executor for "cpu", the CUDA library for "cuda"."""
    from dpm_solver_b200 import ops
    with backend(UniPCOracle() if dev == "cpu" else ops.CudaBackend()):
        yield


def config(**over):
    c = dict(schedule="sd", algo="dpmsolver++", method="multistep", order=2, steps=10, skip_type="time_uniform",
             solver_type="dpmsolver", model_type="noise", cfg=None, lower_order_final=True, denoise_to_zero=False,
             t_end=None, t_start=None, seed=77, thresholding=False, ratio=0.995, max_val=1.0, B=2, shape=(4, 16, 16),
             scale=1.0, channels_last=False, x2_channels_last=False, state_dtype=None, model_dtype=None, guidance="none",
             scales=None, phi=0.0, tuning="auto", sampler="unipc", variant="bh2", use_corrector=True,
             reference_rounding=False)
    c.update(over)
    if c["schedule"] == "flow":
        c.setdefault("shift", 3.0)
        c.setdefault("time_scale", 1000.0)
    return c


def run(s, x, kw):
    """One call on UniPC `s`: kw holds sample()'s arguments plus `variant` (set as an attribute), `thr` (dynamic
    thresholding switched on through correcting_x0_fn, or off) and `inverse`. Returns [y] + intermediates."""
    kw = dict(kw)
    s.variant = kw.pop("variant", "bh2")
    s.correcting_x0_fn = s.dynamic_thresholding_fn if kw.pop("thr", False) else None
    fn = s.inverse if kw.pop("inverse", False) else s.sample
    r = fn(x, **kw)
    return [r[0]] + list(r[1]) if isinstance(r, tuple) else [r]


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert same_bits(a, b), (what, i)


def keyword_sets(thresholding):
    """A base call and calls that differ from it in one or two fields."""
    base = dict(steps=10, order=2, skip_type="time_uniform", lower_order_final=True, t_start=None, t_end=None,
                denoise_to_zero=False, use_corrector=True, return_intermediate=False)
    one = [dict(steps=7), dict(order=3), dict(order=1), dict(use_corrector=False), dict(lower_order_final=False),
           dict(skip_type="logSNR"), dict(skip_type="time_quadratic", order=3), dict(t_start=0.7), dict(t_end=0.02),
           dict(denoise_to_zero=True), dict(return_intermediate=True), dict(inverse=True), dict(variant="bh1"),
           dict(variant="bh1", use_corrector=False, order=3), dict(steps=3, order=3, lower_order_final=False)]
    if thresholding:
        one += [dict(thr=True), dict(thr=True, variant="bh1", return_intermediate=True)]
    return [base] + [dict(base, **d) for d in one]


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("schedule,algo,guidance", [("sd", "dpmsolver++", "float"), ("sd", "dpmsolver", "none"),
                                                    ("flow", "dpmsolver++", "none"), ("flow", "dpmsolver", "float")])
def test_interleaved_configurations(dev, schedule, algo, guidance):
    """~50 calls drawn from the keyword sets, each revisited several times in a seeded order."""
    import dpm_solver_b200 as new
    c = config(schedule=schedule, algo=algo, guidance=guidance, cfg=7.5 if guidance == "float" else None,
               model_type="flow" if schedule == "flow" else "noise")
    kws = keyword_sets(algo == "dpmsolver++")
    with executor(dev):
        rig = FlowRig(new, c, dev)
        s, x = rig.solver(), rig.x()
        rng = random.Random("%s/%s/%s" % (schedule, algo, guidance))
        order = [0, 12, 0, 13, 12, 0] + rng.sample(range(len(kws)), len(kws)) + [rng.randrange(len(kws)) for _ in range(30)]
        fresh = {}
        for n, k in enumerate(order):
            if k not in fresh:
                fresh[k] = run(FlowRig(new, c, dev).solver(), x, kws[k])
                assert all(torch.isfinite(t.float()).all() for t in fresh[k]), kws[k]
            assert_same(run(s, x, kws[k]), fresh[k], (n, kws[k]))
        assert len(fresh) == len(kws) and not s._prep_cache
        # thresholding switched on as an attribute is the solver built with it
        if algo == "dpmsolver++":
            built = FlowRig(new, dict(c, thresholding=True), dev).solver()
            assert_same(run(s, x, dict(kws[0], thr=True)), [built.sample(x, **kws[0])], "built with thresholding")


@pytest.mark.parametrize("dev", DEVICES)
def test_more_configurations_than_the_caches_hold(dev):
    import dpm_solver_b200 as new
    c = config(guidance="float", cfg=7.5)
    with executor(dev):
        rig = FlowRig(new, c, dev)
        s, x = rig.solver(), rig.x()
        sets = [dict(steps=n, order=1 + n % 3, variant=("bh1", "bh2")[n % 2], use_corrector=n % 4 != 1)
                for n in range(5, 25)]
        assert len(sets) > s._CACHE_MAX
        for kw in sets + sets[:3] + sets[::-1]:
            assert_same(run(s, x, kw), run(FlowRig(new, c, dev).solver(), x, kw), kw)
        assert len(s._plan_cache) <= s._CACHE_MAX and len(s._table_cache) <= s._CACHE_MAX


@pytest.mark.parametrize("dev", DEVICES)
def test_schedule_edited_in_place(dev):
    """`_version` of the discrete tables is part of the plan key: an in-place edit is never served a stale plan."""
    import dpm_solver_b200 as new
    c = config(guidance="float", cfg=3.5)
    with executor(dev):
        rig = FlowRig(new, c, dev)
        s, x = rig.solver(), rig.x()
        kw = dict(steps=10, order=3)
        y0 = run(s, x, kw)
        assert_same(run(s, x, kw), y0, "again")
        rig.ns.log_alpha_array.mul_(1.01)
        other = FlowRig(new, c, dev)
        other.ns.log_alpha_array.copy_(rig.ns.log_alpha_array)
        y1 = run(s, x, kw)
        assert_same(y1, run(other.solver(), x, kw), "edited schedule")
        assert not same_bits(y1[0], y0[0])


def shaped_fn(cfg, shapes, dev):
    """model_fn whose network records its input shapes; its conditions have one row, repeated to the batch at hand."""
    import dpm_solver_b200 as new
    from helpers import product_schedule
    ns = product_schedule("sd")

    def net(xx, tt, cc=None):
        shapes.append(tuple(xx.shape))
        one = (-1,) + (1,) * (xx.dim() - 1)
        o = 0.1 * xx.float() + ((tt * 0.001) * 0.05 - 0.02).reshape(one)
        if cc is not None:
            o = o + 0.05 * cc.repeat_interleave(xx.shape[0] // cc.shape[0], 0).reshape(one)
        return o
    if not cfg:
        return new.model_wrapper(lambda xx, tt: net(xx, tt), ns), ns
    return new.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(1, 1, device=dev),
                             unconditional_condition=torch.zeros(1, 1, device=dev), guidance_scale=3.5), ns


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("cfg", [False, True], ids=["plain", "cfg"])
def test_same_numel_other_shape_and_layout(dev, cfg):
    """Inputs of one numel in other shapes, channels_last, row-major again and as a non-dense view: the network sees
    the shape at hand, and the bits are a fresh solver's."""
    import dpm_solver_b200 as new
    base = seeded((4, 4, 16, 16), 5).to(dev)
    big = seeded((4, 4, 16, 32), 6).to(dev)
    inputs = [base, base.reshape(2, 4, 16, 32), base.reshape(8, 2, 16, 16),
              base.contiguous(memory_format=torch.channels_last), base.clone(), big[:, :, :, ::2], base]
    shapes = []
    with executor(dev):
        fn, ns = shaped_fn(cfg, shapes, dev)
        s = new.UniPC(fn, ns, variant="bh2")
        for n, x in enumerate(inputs):
            del shapes[:]
            keep = x.clone()
            y, inter = s.sample(x, steps=8, order=3, return_intermediate=True)
            seen = list(shapes)
            fn2, ns2 = shaped_fn(cfg, [], dev)
            y2, inter2 = new.UniPC(fn2, ns2, variant="bh2").sample(x.clone(), steps=8, order=3, return_intermediate=True)
            rows = (2 if cfg else 1) * x.shape[0]
            assert seen == [(rows,) + tuple(x.shape[1:])] * 8, (n, seen)
            assert y.shape == x.shape, n
            assert_same([y] + inter, [y2] + inter2, n)
            assert same_bits(x, keep), n


@pytest.mark.parametrize("dev", DEVICES)
@pytest.mark.parametrize("guidance", ["none", "float"])
def test_model_fn_shared_with_a_dpm_solver(dev, guidance):
    """One model_fn (whose wrapper caches its conditions by identity and version) serves a long-lived UniPC and a
    long-lived DPM_Solver, called alternately with other arguments: each call equals a fresh solver of its own."""
    import dpm_solver_b200 as new
    c = config(guidance=guidance, cfg=5.0 if guidance == "float" else None)
    calls = [("unipc", dict(steps=10, order=2)), ("dpm", dict(steps=10, order=2)),
             ("unipc", dict(steps=10, order=3, use_corrector=False)), ("dpm", dict(steps=12, order=3)),
             ("dpm", dict(steps=10, order=2, method="singlestep")), ("unipc", dict(steps=10, order=2)),
             ("unipc", dict(steps=7, order=1, denoise_to_zero=True)), ("dpm", dict(steps=10, order=2))]
    with executor(dev):
        rig = FlowRig(new, c, dev)
        x = rig.x()
        uni = rig.solver()
        dpm = new.DPM_Solver(rig.fn, rig.ns, algorithm_type=c["algo"])
        for n, (which, kw) in enumerate(calls * 2):
            other = FlowRig(new, dict(c, sampler=which), dev)
            fresh = other.solver() if which == "unipc" else new.DPM_Solver(other.fn, other.ns, algorithm_type=c["algo"])
            got = (uni if which == "unipc" else dpm).sample(x, **kw)
            assert same_bits(got, fresh.sample(x, **kw)), (n, which, kw)


# ---- device only -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("schedule", ["sd", "flow"])
def test_steady_state_call_reads_nothing_back(schedule):
    """A cached configuration on the long-lived solver runs without a host synchronisation, with the same bits."""
    import dpm_solver_b200 as new
    c = config(schedule=schedule, model_type="flow" if schedule == "flow" else "noise", guidance="float", cfg=4.0,
               thresholding=True)
    with executor("cuda"):
        rig = FlowRig(new, c, "cuda")
        s, x = rig.solver(), rig.x()
        for kw in (dict(steps=10, order=3), dict(steps=8, order=2, use_corrector=False), dict(steps=10, order=3)):
            want = s.sample(x, **kw)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                got = s.sample(x, **kw)
            finally:
                torch.cuda.set_sync_debug_mode("default")
            assert same_bits(got, want), kw


@pytest.mark.gpu
def test_diffedit_corrector_reuse():
    """One DiffEditCorrector as UniPC's `correcting_xt_fn` across runs that map step k to other times (other `steps`,
    `t_end`, `denoise_to_zero`, which calls it at step + 1, another `time_fn`, other orders): every run equals the
    numpy executor driving the notebook's corrector_fn -- x*mask + (1 - mask)*(alpha*x0 + sigma*noise), with the
    normals torch.randn draws from the same generator state -- and a steady-state run reads nothing back."""
    import dpm_solver_b200 as new
    c = config(B=2)
    x0 = seeded((2, 4, 16, 16), 21)
    mask = (seeded((16, 16), 22) > 0).float()
    gen, gen_ref = torch.Generator("cuda"), torch.Generator("cuda")
    time_fns = {"identity": None, "shrunk": lambda t: t * 0.75 + 0.001}
    now = {"time_fn": None}
    with executor("cpu"):
        cpu_rig = FlowRig(new, c, "cpu")

        def corrector_fn(xt, t, step):      # diffedit_inpaint.ipynb
            te = t if now["time_fn"] is None else now["time_fn"](t)
            te = te.reshape(-1)[:1]
            noise = torch.randn((1, *x0.shape), device="cuda", generator=gen_ref).cpu()[0]
            al, sg = cpu_rig.ns.marginal_alpha(te), cpu_rig.ns.marginal_std(te)
            inter = al * x0 + sg * noise
            return xt * mask + (1 - mask) * inter

        cpu_solver = new.UniPC(cpu_rig.fn, cpu_rig.ns, correcting_xt_fn=corrector_fn)
    with executor("cuda"):
        rig = FlowRig(new, c, "cuda")
        x = rig.x()
        corr = new.DiffEditCorrector(rig.ns, x0.cuda(), mask.cuda(), generator=gen)
        s = new.UniPC(rig.fn, rig.ns, correcting_xt_fn=corr)
    runs = [("identity", dict(steps=10, order=2)), ("identity", dict(steps=15, order=2)),
            ("identity", dict(steps=10, order=2, t_end=0.05)), ("identity", dict(steps=10, order=2, denoise_to_zero=True)),
            ("shrunk", dict(steps=10, order=2)), ("identity", dict(steps=10, order=2)),
            ("identity", dict(steps=9, order=3, use_corrector=False)), ("identity", dict(steps=9, order=1))]
    for n, (name, kw) in enumerate(runs):
        corr.time_fn = now["time_fn"] = time_fns[name]
        gen.manual_seed(100 + n), gen_ref.manual_seed(100 + n)
        with executor("cuda"):
            got = run(s, x, dict(kw, return_intermediate=True))
        with executor("cpu"):
            want = run(cpu_solver, cpu_rig.x(), dict(kw, return_intermediate=True))
        assert_same(got, want, (n, name, kw))
    # the first configuration once more: every label is cached, nothing is read back
    corr.time_fn = now["time_fn"] = None
    gen.manual_seed(100), gen_ref.manual_seed(100)
    with executor("cpu"):
        want = run(cpu_solver, cpu_rig.x(), runs[0][1])
    with executor("cuda"):
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            got = s.sample(x, **runs[0][1])
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert_same([got], want, "steady state")
