"""One long-lived `DPM_Solver` serving whatever arrives: other sampling arguments, other shapes with the same numel,
other layouts and dtypes, more configurations than its caches hold, a schedule edited in place, attributes changed
between calls, and one `DiffEditCorrector` across configurations. Invariant throughout: a call on the long-lived solver
returns exactly the bits a fresh solver returns for that call (device against device, so it holds for the adaptive
method too), with spot checks of the same against the unmodified reference on CPU."""
import contextlib
import io
import random

import pytest
import torch

from cases import seeded
from gpu_configs import Rig, reference, same_bits
from oracle import ref_loader

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def config(**over):
    c = dict(schedule="sd", algo="dpmsolver++", method="multistep", order=2, steps=12, skip_type="time_uniform",
             solver_type="dpmsolver", model_type="noise", cfg=None, lower_order_final=True, denoise_to_zero=False,
             t_end=None, t_start=None, seed=77, thresholding=False, ratio=0.995, max_val=1.0, B=4, shape=(4, 16, 16),
             scale=1.0, channels_last=False, x2_channels_last=False, state_dtype=None, model_dtype=None, guidance="none",
             scales=None, phi=0.0, tuning="auto")
    c.update(over)
    return c


def call(s, x, **kw):
    """sample() -> list of tensors (y, then the intermediates when asked for); the adaptive method prints."""
    with contextlib.redirect_stdout(io.StringIO()):
        r = s.sample(x, **kw)
    return [r[0]] + list(r[1]) if isinstance(r, tuple) else [r]


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for i, (a, b) in enumerate(zip(got, want)):
        assert same_bits(a, b), (what, i)


# ---- other sampling arguments --------------------------------------------------------------------------------------
def keyword_sets(t_end):
    """A base call and eleven that differ from it in one field."""
    base = dict(steps=12, order=2, skip_type="time_uniform", method="multistep", solver_type="dpmsolver",
                lower_order_final=True, t_start=None, t_end=t_end, denoise_to_zero=False, return_intermediate=False)
    one = [dict(steps=7), dict(order=3), dict(order=1), dict(skip_type="logSNR"), dict(method="singlestep"),
           dict(method="adaptive", atol=0.05, rtol=0.2), dict(solver_type="taylor"), dict(lower_order_final=False, steps=8),
           dict(t_start=0.7), dict(t_end=0.02), dict(denoise_to_zero=True), dict(return_intermediate=True)]
    return [base] + [dict(base, **d) for d in one]


@pytest.mark.parametrize("guidance", ["none", "float", "per_sample", "multi"])
@pytest.mark.parametrize("algo", ["dpmsolver++", "dpmsolver"])
@pytest.mark.parametrize("schedule", ["sd", "vp_linear"])
def test_interleaved_configurations(cuda_backend, schedule, algo, guidance):
    """~60 calls drawn from 13 keyword sets, each revisited several times in a seeded order."""
    import dpm_solver_b200 as new
    c = config(schedule=schedule, algo=algo, guidance=guidance, cfg=7.5 if guidance == "float" else None,
               scales={"per_sample": [7.5, 1.0, 0.0, -2.0], "multi": [4.0, -1.5]}.get(guidance))
    kws = keyword_sets(1e-3 if schedule == "vp_linear" else None)
    rig = Rig(new, c, DEV)
    s, x = rig.solver(), rig.x()
    rng = random.Random("%s/%s/%s" % (schedule, algo, guidance))
    order = [0, 1, 0, 2, 1, 0] + rng.sample(range(len(kws)), len(kws)) + [rng.randrange(len(kws)) for _ in range(41)]
    fresh = {}
    for n, k in enumerate(order):
        if k not in fresh:
            other = Rig(new, c, DEV)
            fresh[k] = call(other.solver(), x, **kws[k])
            assert all(torch.isfinite(t.float()).all() for t in fresh[k]), kws[k]
        assert_same(call(s, x, **kws[k]), fresh[k], (n, kws[k]))
    assert len(fresh) == len(kws)
    assert s._prep_cache or guidance in ("per_sample", "multi")     # (those two read per-launch data: never frozen)
    if ref_loader.available() and guidance in ("none", "float"):
        ref_rig = Rig(reference(), c)
        for k, kw in enumerate(kws):
            if kw["method"] != "adaptive":
                assert_same(fresh[k], call(ref_rig.solver(), ref_rig.x(), **kw), ("reference", kw))


# ---- other shapes, layouts and dtypes ------------------------------------------------------------------------------
def shaped_fn(cfg, shapes, out_dtype=lambda: None):
    """model_fn whose network records its input shapes; its conditions have one row, repeated to the batch at hand, so
    that one wrapper serves every batch size."""
    import dpm_solver_b200 as new
    from helpers import product_schedule
    ns = product_schedule("sd")

    def net(xx, tt, cc=None):
        shapes.append(tuple(xx.shape))
        one = (-1,) + (1,) * (xx.dim() - 1)
        o = 0.1 * xx.float() + ((tt * 0.001) * 0.05 - 0.02).reshape(one)
        if cc is not None:
            o = o + 0.05 * cc.repeat_interleave(xx.shape[0] // cc.shape[0], 0).reshape(one)
        return o if out_dtype() is None else o.to(out_dtype())
    if not cfg:
        return new.model_wrapper(lambda xx, tt: net(xx, tt), ns), ns
    return new.model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(1, 1, device=DEV),
                             unconditional_condition=torch.zeros(1, 1, device=DEV), guidance_scale=3.5), ns


def layout_class(t):
    return "row-major" if t.is_contiguous() else "channels_last" if t.is_contiguous(memory_format=torch.channels_last) \
        else "other"


@pytest.mark.parametrize("cfg", [False, True], ids=["plain", "cfg"])
def test_same_numel_other_shape_and_layout(cuda_backend, cfg):
    """Inputs of one numel in other shapes, channels_last, row-major again and as a non-dense view: shape, layout class
    and bits of a fresh solver's result, and the network saw the shape at hand every time."""
    import dpm_solver_b200 as new
    base = seeded((4, 4, 16, 16), 5).to(DEV)
    big = seeded((4, 4, 16, 32), 6).to(DEV)
    inputs = [base, base.reshape(2, 4, 16, 32), base.reshape(8, 2, 16, 16),
              base.contiguous(memory_format=torch.channels_last), base.clone(), big[:, :, :, ::2], base]
    shapes = []
    fn, ns = shaped_fn(cfg, shapes)
    s = new.DPM_Solver(fn, ns)
    for n, x in enumerate(inputs):
        del shapes[:]
        keep = x.clone()
        y, inter = s.sample(x, steps=8, order=2, return_intermediate=True)
        seen = list(shapes)
        fn2, ns2 = shaped_fn(cfg, [])
        y2, inter2 = new.DPM_Solver(fn2, ns2).sample(x.clone(), steps=8, order=2, return_intermediate=True)
        rows = (2 if cfg else 1) * x.shape[0]
        assert seen == [(rows,) + tuple(x.shape[1:])] * 8, (n, seen)
        assert y.shape == x.shape and layout_class(y) == layout_class(y2) != "other", n
        if layout_class(x) != "other":
            assert layout_class(y) == layout_class(x), n        # dense layouts are kept end to end (DESIGN section 3)
        assert_same([y] + inter, [y2] + inter2, n)
        assert same_bits(x, keep), n
    assert s._prep_cache


def test_other_dtype_after_prepared(cuda_backend):
    """fp32 x, a bf16 x in the reference's promotion mode, fp32 again, while the network's output type changes from
    one sequence of calls to the next: never a launch frozen for the other type."""
    import dpm_solver_b200 as new
    out = [None]
    fn, ns = shaped_fn(True, [], lambda: out[0])
    s = new.DPM_Solver(fn, ns)
    x = seeded((4, 4, 16, 16), 8).to(DEV)
    for n, (xin, md) in enumerate([(x, None), (x, None), (x.bfloat16(), None), (x, None), (x, torch.bfloat16),
                                   (x, torch.bfloat16), (x, None), (x.bfloat16(), torch.bfloat16), (x, None)]):
        out[0] = md
        y = s.sample(xin, steps=9, order=3)
        fn2, ns2 = shaped_fn(True, [], lambda: md)
        y2 = new.DPM_Solver(fn2, ns2).sample(xin.clone(), steps=9, order=3)
        assert y.dtype == torch.float32 and same_bits(y, y2), n
    assert s._prep_cache


# ---- cache bounds ---------------------------------------------------------------------------------------------------
def test_more_configurations_than_the_plan_and_table_caches_hold(cuda_backend):
    import dpm_solver_b200 as new
    rig = Rig(new, config(guidance="float", cfg=7.5), DEV)
    s, x = rig.solver(), rig.x()
    sets = [dict(steps=n, order=2 + n % 2) for n in range(5, 25)]
    assert len(sets) > s._CACHE_MAX
    fresh = []
    for kw in sets + sets[:3] + sets[::-1]:
        got = call(s, x, **kw)
        fresh.append(call(Rig(new, rig.c, DEV).solver(), x, **kw))
        assert_same(got, fresh[-1], kw)
    assert len(s._plan_cache) <= s._CACHE_MAX and len(s._table_cache) <= s._CACHE_MAX


def test_prepared_launch_cache_is_cleared_in_the_middle_of_a_call(cuda_backend):
    """Distinct (steps, batch) pairs until the 512-entry bound of `_prep_cache` falls inside a sample() call, then
    every earlier call again."""
    import dpm_solver_b200 as new
    rig = Rig(new, config(), DEV)
    s = rig.solver()
    xs = {B: seeded((B, 4, 16, 16), B).to(DEV) for B in (1, 2, 3, 4)}
    done, crossed = [], None
    for steps in range(30, 60):
        for B in xs:
            before = len(s._prep_cache)
            got = call(s, xs[B], steps=steps, order=2)
            want = call(Rig(new, rig.c, DEV).solver(), xs[B], steps=steps, order=2)
            assert_same(got, want, (steps, B))
            done.append((steps, B, want))
            if len(s._prep_cache) < before:
                crossed = (before, steps)
                break
        if crossed:
            break
    assert crossed and 0 < 512 - crossed[0] < crossed[1], crossed       # the bound fell inside the run
    for steps, B, want in done:
        assert_same(call(s, xs[B], steps=steps, order=2), want, ("again", steps, B))
        assert_same(call(s, xs[B], steps=steps, order=2), want, ("prepared again", steps, B))


def test_schedule_edited_in_place_after_prepared_launches(cuda_backend):
    """`_version` of the tables is part of the plan id: an in-place edit never meets the frozen launches' scalars."""
    import dpm_solver_b200 as new
    rig = Rig(new, config(guidance="float", cfg=3.5), DEV)
    s, x = rig.solver(), rig.x()
    y0 = call(s, x, steps=10, order=2)
    assert_same(call(s, x, steps=10, order=2), y0, "prepared")
    assert s._prep_cache
    rig.ns.log_alpha_array.mul_(1.01)
    other = Rig(new, rig.c, DEV)
    other.ns.log_alpha_array.copy_(rig.ns.log_alpha_array)
    y1 = call(s, x, steps=10, order=2)
    assert_same(y1, call(other.solver(), x, steps=10, order=2), "edited schedule")
    assert not same_bits(y1[0], y0[0])


def test_device_coefficients_are_never_frozen(cuda_backend):
    """A launch that reads its scalars from a device block is not one PreparedStep may freeze: the descriptor would
    keep a pointer into a block it does not own."""
    from dpm_solver_b200 import ops
    x = seeded((2, 4, 8, 8), 1).to(DEV)
    a = ops.StepArgs(form=ops.FORM_LIN1, n_model=0, x=x, m0=x.clone(), a=1.0, c0=0.5, state_dtype=torch.float32)
    assert cuda_backend.prepare(a) is not None
    a.coef_dev = torch.zeros(16, device=DEV)
    assert cuda_backend.prepare(a) is None


# ---- attributes changed between calls ------------------------------------------------------------------------------
def test_changed_solver_attributes(cuda_backend):
    """`thresholding_max_val`, `dynamic_thresholding_ratio` and `correcting_x0_fn` are read at every call, and a
    per-sample `guidance_scale` tensor is read on the device at every launch: a call after the change equals a fresh
    solver built with the new values."""
    import dpm_solver_b200 as new
    c = config(schedule="ddpm_linear", guidance="per_sample", scales=[7.5, 1.0, 0.0, -2.0], thresholding=True, scale=3.0)
    rig = Rig(new, c, DEV)
    s, x = rig.solver(), rig.x()
    kw = dict(steps=10, order=2)

    def fresh(hook="keep", **over):
        r = Rig(new, dict(c, **over), DEV)
        f = r.solver()
        if hook != "keep":
            f = r.mod.DPM_Solver(r.fn, r.ns, algorithm_type=c["algo"], correcting_x0_fn=hook)
        return call(f, x, **kw)

    assert_same(call(s, x, **kw), fresh(), "as built")
    s.thresholding_max_val = 0.5
    assert_same(call(s, x, **kw), fresh(max_val=0.5), "thresholding_max_val")
    s.dynamic_thresholding_ratio = 0.9
    assert_same(call(s, x, **kw), fresh(max_val=0.5, ratio=0.9), "dynamic_thresholding_ratio")
    rig.scale.copy_(torch.tensor([0.0, 3.5, 7.5, 1.0]))
    assert_same(call(s, x, **kw), fresh(max_val=0.5, ratio=0.9, scales=[0.0, 3.5, 7.5, 1.0]), "scales written in place")

    # correcting_x0_fn: none (launches get frozen) -> the solver's own thresholding -> a python hook -> none again
    rig = Rig(new, config(schedule="ddpm_linear", guidance="float", cfg=3.5, scale=3.0), DEV)
    s, x = rig.solver(), rig.x()
    c = rig.c
    none = call(s, x, **kw)
    assert_same(call(s, x, **kw), none, "prepared")
    assert s._prep_cache
    s.correcting_x0_fn = s.dynamic_thresholding_fn
    thr = call(s, x, **kw)
    assert_same(thr, fresh(thresholding=True), "dynamic thresholding switched on")
    assert not same_bits(thr[0], none[0])
    hook = lambda x0, t: x0.clamp(-0.8, 0.8)
    s.correcting_x0_fn = hook
    assert_same(call(s, x, **kw), fresh(hook=hook), "python hook")
    s.correcting_x0_fn = None
    assert_same(call(s, x, **kw), none, "back to none")


def test_two_devices(cuda_backend):
    """cuda:0 and cuda:1 inputs alternate on one solver; the current device stays 0."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two devices")
    import dpm_solver_b200 as new
    fn, ns = shaped_fn(False, [])
    s = new.DPM_Solver(fn, ns)
    x = seeded((4, 4, 16, 16), 3)
    want = None
    for dev in ("cuda:0", "cuda:1", "cuda:0", "cuda:1", "cuda:1", "cuda:0"):
        y = s.sample(x.to(dev), steps=8, order=2)
        assert y.device == torch.device(dev) and torch.cuda.current_device() == 0
        want = y.cpu() if want is None else want
        assert same_bits(y, want), dev


# ---- one DiffEdit corrector across configurations ------------------------------------------------------------------
@pytest.mark.skipif(not ref_loader.available(), reason="oracle/_ref not built and no reference tree")
def test_diffedit_corrector_reuse(cuda_backend):
    """One DiffEditCorrector, held by one solver as `correcting_xt_fn`, across configurations that map step k to other
    times (other `steps`, other `t_end`, `denoise_to_zero`, which calls it at step + 1, another `time_fn`): every run
    equals the unmodified reference on CPU driving the notebook's corrector_fn, composed from the reference's own
    add_noise with the normals torch.randn draws from the same generator state. A steady-state run reads nothing back
    from the device."""
    import dpm_solver_b200 as new
    ref = reference()
    c = config(B=2)
    rig, ref_rig = Rig(new, c, DEV), Rig(ref, c)
    x, x0 = rig.x(), seeded((2, 4, 16, 16), 21)
    mask = (seeded((16, 16), 22) > 0).float()
    gen, gen_ref = torch.Generator(DEV), torch.Generator(DEV)
    time_fns = {"identity": None, "shrunk": lambda t: t * 0.75 + 0.001}
    corr = new.DiffEditCorrector(rig.ns, x0.to(DEV), mask.to(DEV), generator=gen)
    s = new.DPM_Solver(rig.fn, rig.ns, correcting_xt_fn=corr)
    now = {"time_fn": None}

    def corrector_fn(xt, t, step):      # diffedit_inpaint.ipynb, on the reference's add_noise
        te = t if now["time_fn"] is None else now["time_fn"](t)
        noise = torch.randn((1, *x0.shape), device=DEV, generator=gen_ref).cpu()
        inter = ref_solver.add_noise(x0, te.reshape(-1)[:1], noise=noise)
        return xt * mask + (1 - mask) * inter

    ref_solver = ref.DPM_Solver(ref_rig.fn, ref_rig.ns, correcting_xt_fn=corrector_fn)
    runs = [("identity", dict(steps=10, order=2)), ("identity", dict(steps=15, order=2)),
            ("identity", dict(steps=10, order=2, t_end=0.05)), ("identity", dict(steps=10, order=2, denoise_to_zero=True)),
            ("shrunk", dict(steps=10, order=2)), ("identity", dict(steps=10, order=2)),
            ("identity", dict(steps=9, order=3, method="singlestep"))]
    for n, (name, kw) in enumerate(runs):
        corr.time_fn = now["time_fn"] = time_fns[name]
        gen.manual_seed(100 + n), gen_ref.manual_seed(100 + n)
        got = call(s, x, return_intermediate=True, **kw)
        want = call(ref_solver, ref_rig.x(), return_intermediate=True, **kw)
        assert_same(got, want, (n, name, kw))
    # the first configuration once more: every label is cached, nothing is read back
    corr.time_fn = now["time_fn"] = None
    gen.manual_seed(100), gen_ref.manual_seed(100)
    want = call(ref_solver, ref_rig.x(), **runs[0][1])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = s.sample(x, **runs[0][1])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert_same([got], want, "steady state")
    with pytest.raises(ValueError):
        new.DiffEditCorrector(rig.ns, x0.to(DEV), mask.to(DEV), generator=torch.Generator())(x, torch.tensor(0.5, device=DEV), 0)


# ---- the adaptive solver's surplus network evaluations ------------------------------------------------------------
@pytest.mark.skipif(not ref_loader.available(), reason="oracle/_ref not built and no reference tree")
@pytest.mark.xfail(strict=True, reason="the device controller still runs the iterations of a chunk enqueued after `done`")
def test_adaptive_network_calls_equal_the_reference_nfe(cuda_backend):
    import dpm_solver_b200 as new
    counts = []
    for order in (2, 3):
        for atol, rtol in ((0.05, 0.2), (0.0078, 0.05), (0.02, 0.1)):
            c = config(method="adaptive", order=order, algo="dpmsolver", B=2)
            rig, ref_rig = Rig(new, c, DEV), Rig(reference(), c)
            kw = dict(method="adaptive", order=order, atol=atol, rtol=rtol)
            rig.calls, ref_rig.calls = [], []
            call(rig.solver(), rig.x(), **kw), call(ref_rig.solver(), ref_rig.x(), **kw)
            counts.append((len(rig.calls), len(ref_rig.calls)))
    assert all(a == b for a, b in counts), counts
