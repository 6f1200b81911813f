"""One long-lived solver per feature (TCFG, frequency-decoupled guidance) on the H100, under the invariant of
tests/test_gpu_solver_reuse.py: every call returns the bits a fresh wrapper and solver return for that call.

FDG: between calls x switches between row-major and channels_last and between two shapes of one size, every tensor form
of fdg_scales is edited in place, sample() alternates with inverse() under other steps, orders and t_end, and dynamic
thresholding is switched on and off; once under multistep order 2, whose frozen steps (`PreparedStep`s holding the one
output g) are served across those changes, and once under UniPC. TCFG: a per-sample scale tensor edited in place across
layouts and model dtypes, a one-element scale tensor set to 1 (the bypass: B network rows, not 2B) and back, `tcfg`
switched off and on on one wrapper, and a run stopped by an exception the network raises."""
import pytest
import torch

from gpu_configs import same_bits
from test_gpu_random_configs import LaunchSpy
from test_tcfg import product_schedule

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = 3
S1, S2 = (B, 4, 24, 24), (B, 9, 16, 16)     # one size per sample; both planes take levels = 3
ROWS = [[6.0, 3.0, 1.5], [2.0, 4.0, 1.0], [1.0, 1.0, 5.0]]


class Boom(RuntimeError):
    pass


def make_net(dtype=None, raise_at=None):
    """Products and sums only, outputs in dtype[0] when set (the network's own dtype, switchable between calls); raises
    Boom at its call number raise_at[0] (1-based) when set, counting in raise_at[1]."""
    def net(x, t, c):
        if raise_at is not None:
            raise_at[1] += 1
            if raise_at[1] == raise_at[0]:
                raise Boom("network call %d" % raise_at[1])
        cc = c.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
        tt = t.reshape((-1,) + (1,) * (x.dim() - 1)).to(x.dtype)
        o = 0.45 * x + 0.05 * cc * x * x - 0.1 + 0.05 * cc + 1e-4 * tt
        return o if dtype is None or dtype[0] is None else o.to(dtype[0])
    return net


def xs(seed, shape=S1, cl=False):
    x = torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(DEV)
    return x.contiguous(memory_format=torch.channels_last) if cl else x


def wrapper(ns, net=None, **kw):
    import dpm_solver_b200 as new
    return new.model_wrapper(net or make_net(), ns, model_type="noise", guidance_type="classifier-free",
                             condition=torch.ones(B, 1, device=DEV), unconditional_condition=torch.zeros(B, 1, device=DEV),
                             **kw)


def solver(fn, ns, kind, thr=False):
    """A DPM_Solver or UniPC on `fn`; `thr` switches dynamic thresholding on through correcting_x0_fn, as a user would
    on a live solver."""
    import dpm_solver_b200 as new
    s = new.UniPC(fn, ns, variant="bh2") if kind == "unipc" else new.DPM_Solver(fn, ns)
    set_thresholding(s, thr)
    return s


def set_thresholding(s, thr):
    s.correcting_x0_fn = s.dynamic_thresholding_fn if thr else None


def run(s, x, inverse=False, **skw):
    return (s.inverse if inverse else s.sample)(x, **skw)


# ---- frequency-decoupled guidance ------------------------------------------------------------------------------------

def fdg_scales(form):
    if form == "vec":
        return torch.tensor(ROWS[0], device=DEV)
    if form == "listed":
        return [torch.tensor(v, device=DEV) for v in ROWS[0]]
    if form == "converted":
        return torch.tensor(ROWS, dtype=torch.bfloat16, device=DEV)
    return torch.tensor(ROWS, device=DEV)                  # in place: fp32 [B, N] on the device


def edit_fdg(form, w, k):
    """The k-th in-place edit: one listed tensor at a time, or the whole tensor (values stay exact in bf16)."""
    if form == "listed":
        w[k % 3].mul_(-0.5).add_(1.25)
    else:
        w.mul_(-0.5).add_(1.25 + 0.25 * k)


def clone_fdg(w):
    return [t.clone() for t in w] if isinstance(w, list) else w.clone()


# (seed, shape, channels_last, inverse, sampling arguments, thresholding, edit before the call); an edit is followed by
# a call of the previous call's shape and layout, so that only the tensors' versions tell the two apart
FDG_CALLS = [(1, S1, False, False, dict(steps=6), False, False),
             (1, S1, False, False, dict(steps=6), False, False),
             (2, S1, True, False, dict(steps=6), False, False),
             (2, S1, True, False, dict(steps=6), False, True),
             (3, S2, False, True, dict(steps=5), False, False),
             (3, S2, False, True, dict(steps=5), False, True),
             (4, S2, False, False, dict(steps=6, t_end=0.05), True, False),
             (4, S2, False, False, dict(steps=6, t_end=0.05), True, True),
             (5, S1, False, False, dict(steps=7, order=3), False, False),
             (5, S1, False, False, dict(steps=7, order=3), False, True),
             (6, S2, True, False, dict(steps=6), True, True),
             (6, S1, False, False, dict(steps=6), False, True),
             (7, S1, False, True, dict(steps=4, order=1), False, True)]


@pytest.mark.parametrize("form", ["vec", "listed", "converted", "in_place"])
@pytest.mark.parametrize("kind", ["dpm", "unipc"])
def test_fdg_solver_across_calls(cuda_backend, kind, form):
    ns = product_schedule("noise")
    w = fdg_scales(form)
    fn = wrapper(ns, fdg_scales=w)
    s = solver(fn, ns, kind)
    served = 0
    for i, (seed, shape, cl, inverse, skw, thr, edit) in enumerate(FDG_CALLS):
        if inverse and kind == "unipc":
            continue                                        # (UniPC has no inverse())
        if edit:
            edit_fdg(form, w, i)
        skw = dict(dict(order=2, method="multistep") if kind == "dpm" else dict(order=2), **skw)
        set_thresholding(s, thr)
        x = xs(seed, shape, cl)
        with LaunchSpy() as spy:
            got = run(s, x, inverse, **skw)
        served += spy.plain + spy.dup
        fresh = solver(wrapper(ns, fdg_scales=clone_fdg(w)), ns, kind, thr)
        assert same_bits(got, run(fresh, x.clone(), inverse, **skw)), (i, shape, cl, inverse, skw, thr)
    if kind == "dpm":
        assert served, "no frozen FDG step was served"


# ---- TCFG ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["dpm", "unipc"])
def test_tcfg_scale_edits_layouts_and_model_dtypes(cuda_backend, kind):
    """A per-sample scale tensor (DPM_Solver; UniPC takes one scale: a one-element tensor) edited in place, x switched
    between row-major and channels_last and the network's output dtype between fp32, bf16 and fp16."""
    ns = product_schedule("noise")
    w = torch.tensor([4.5, 1.0, 2.5], device=DEV) if kind == "dpm" else torch.tensor([4.5], device=DEV)
    md = [None]
    s = solver(wrapper(ns, net=make_net(md), guidance_scale=w, tcfg=True), ns, kind)
    edits = [None, lambda: w.mul_(-1.0).add_(2.0), None, lambda: w.add_(0.5), None, lambda: w.fill_(3.0)]
    for i, edit in enumerate(edits):
        if edit is not None:
            edit()
        for cl, dt in ((False, None), (True, torch.bfloat16), (True, None), (False, torch.float16)):
            md[0] = dt
            x = xs(20 + i, cl=cl)
            skw = dict(steps=6, order=2 if cl else 3)
            got = s.sample(x, **skw)
            fresh = solver(wrapper(ns, net=make_net([dt]), guidance_scale=w.clone(), tcfg=True), ns, kind)
            assert same_bits(got, fresh.sample(x.clone(), **skw)), (i, cl, dt)


@pytest.mark.parametrize("kind", ["dpm", "unipc"])
def test_tcfg_one_scale_tensor_edited_to_one_and_back(cuda_backend, kind):
    """A one-element scale tensor set to 1 in place bypasses the halves (the network gets B rows, not 2B) and set back
    combines them again: the model-input time rows of the solver's cached tables must follow. Every run,
    denoise_to_zero included, is a fresh solver's."""
    ns = product_schedule("flow")
    w = torch.tensor([4.5], device=DEV)
    import dpm_solver_b200 as new
    mk = (lambda f: new.UniPC(f, ns)) if kind == "unipc" else (lambda f: new.DPM_Solver(f, ns))
    wrap = lambda scale: new.model_wrapper(make_net(), ns, model_type="flow", guidance_type="classifier-free",
                                           condition=torch.ones(B, 1, device=DEV),
                                           unconditional_condition=torch.zeros(B, 1, device=DEV),
                                           guidance_scale=scale, tcfg=True)
    s = mk(wrap(w))
    for i, v in enumerate([4.5, 1.0, 3.0, 1.0, 1.0, 2.0]):
        w.fill_(v)
        x = xs(50 + i)
        skw = dict(steps=5, order=2, denoise_to_zero=i >= 4)
        assert same_bits(s.sample(x, **skw), mk(wrap(w.clone())).sample(x.clone(), **skw)), (i, v)


def test_tcfg_switched_off_and_on(cuda_backend):
    """`tcfg` switched on one wrapper: plain CFG and TCFG on the same cached plans and frozen steps (the PreparedStep key
    carries raw.tcfg), thresholding now and then, sample() and inverse()."""
    ns = product_schedule("noise")
    fn = wrapper(ns, guidance_scale=4.5, tcfg=False)
    s = solver(fn, ns, "dpm")
    calls = [(False, dict(steps=6, order=2), False, None), (False, dict(steps=6, order=2), False, True),
             (False, dict(steps=6, order=2), False, False), (False, dict(steps=6, order=2), False, True),
             (True, dict(steps=5, order=2), False, False), (True, dict(steps=5, order=2), False, True),
             (False, dict(steps=7, order=3), True, None), (False, dict(steps=7, order=3), True, False),
             (False, dict(steps=7, order=1, t_end=0.05), False, True), (False, dict(steps=7, order=1, t_end=0.05),
                                                                       False, False)]
    for i, (inverse, skw, thr, tc) in enumerate(calls):
        if tc is not None:
            fn.tcfg = tc
        set_thresholding(s, thr)
        x = xs(60 + i % 3)
        got = run(s, x, inverse, **skw)
        fresh = solver(wrapper(ns, guidance_scale=4.5, tcfg=fn.tcfg), ns, "dpm", thr)
        assert same_bits(got, run(fresh, x.clone(), inverse, **skw)), (i, inverse, skw, thr, fn.tcfg)


@pytest.mark.parametrize("kind", ["dpm", "unipc"])
@pytest.mark.parametrize("k", [1, 3])
def test_tcfg_run_stopped_by_the_network(cuda_backend, kind, k):
    """The network raises at its call k of a TCFG run; the next run and a direct data_prediction_fn call are a fresh
    solver's."""
    ns = product_schedule("noise")
    plan = [None, 0]
    w = torch.tensor([4.5, 1.0, 2.5], device=DEV) if kind == "dpm" else 4.5
    s = solver(wrapper(ns, net=make_net(raise_at=plan), guidance_scale=w, tcfg=True), ns, kind)
    x, x2 = xs(30, cl=True), xs(31)
    plan[:] = [k, 0]
    with pytest.raises(Boom):
        s.sample(x, steps=6, order=2)
    plan[:] = [None, 0]
    fresh = lambda: solver(wrapper(ns, guidance_scale=w, tcfg=True), ns, kind)
    t = torch.full((B,), 0.5, device=DEV)
    assert same_bits(s.data_prediction_fn(x2, t), fresh().data_prediction_fn(x2.clone(), t))
    assert same_bits(s.sample(x2, steps=6, order=2), fresh().sample(x2.clone(), steps=6, order=2))
    assert same_bits(s.sample(x, steps=6, order=2), fresh().sample(x.clone(), steps=6, order=2))
