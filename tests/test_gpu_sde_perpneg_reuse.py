"""One long-lived SDE-DPM-Solver++ solver and long-lived Perp-Neg wrappers on the H100, under the invariant of
tests/test_gpu_solver_reuse.py: every call returns the bits a fresh wrapper and solver return for that call, from the
same generator state.

SDE: between calls eta goes 0 -> 1 -> 0.5 -> 0 with an explicit generator and then with None (the device's default
generator), the order and steps change, x switches between two shapes of one size and between row-major and
channels_last, the state between fp32 and bf16, and dynamic thresholding is switched on and off through
correcting_x0_fn; a capture() sits in the middle of the sequence, and one run is stopped by an exception the network
raises, after which the generator sits where the contract's draws of the finished updates leave it.

Perp-Neg: a K = 2 and a K = 4 wrapper on one schedule, each with one solver; their scales are switched between calls,
x changes values, shape and layout, the network's output dtype changes, and an adaptive run is followed by multistep
runs."""
import pytest
import torch

from gpu_configs import same_bits

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = 3
S1, S2 = (B, 4, 24, 24), (B, 9, 16, 16)     # one size per sample
BF = torch.bfloat16


class Boom(RuntimeError):
    pass


def make_net(dtype=None, raise_at=None):
    """Products and sums only (the same bits on every device), outputs in dtype[0] when set; raises Boom at its call
    number raise_at[0] (1-based) when set, counting in raise_at[1]."""
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


def schedule():
    import dpm_solver_b200 as new
    return new.NoiseScheduleVP("discrete", betas=torch.linspace(1e-4, 2e-2, 1000))


def set_thresholding(s, thr):
    s.correcting_x0_fn = s.dynamic_thresholding_fn if thr else None


# ---- SDE-DPM-Solver++ ------------------------------------------------------------------------------------------------

def sde_wrapper(ns, net=None):
    import dpm_solver_b200 as new
    return new.model_wrapper(net or make_net(), ns, model_type="noise", guidance_type="classifier-free",
                             condition=torch.ones(B, 1, device=DEV),
                             unconditional_condition=torch.zeros(B, 1, device=DEV), guidance_scale=3.5)


def sde_solver(fn, ns, state_dtype=None, thr=False):
    import dpm_solver_b200 as new
    s = new.DPM_Solver(fn, ns, algorithm_type="sde-dpmsolver++", state_dtype=state_dtype)
    set_thresholding(s, thr)
    return s


def generator(kind, seed):
    """("g": an explicit CUDA generator, None: the default one) seeded with `seed`; returns (argument, generator)."""
    if kind == "g":
        g = torch.Generator(DEV).manual_seed(seed)
        return g, g
    torch.cuda.manual_seed(seed)
    return None, torch.cuda.default_generators[torch.cuda.current_device()]


# (eta, generator, order, steps, shape, channels_last, state dtype, thresholding)
SDE_CALLS = [(0.0, "g", 2, 5, S1, False, None, False),
             (1.0, "g", 2, 6, S1, True, None, True),
             "capture",
             (0.5, "g", 3, 7, S2, False, BF, False),
             (0.0, "g", 1, 4, S2, True, None, True),
             "capture",
             (0.0, None, 3, 6, S1, False, BF, True),
             (1.0, None, 2, 5, S2, True, None, False),
             "capture",
             (1.0, None, 2, 5, S2, True, None, False),
             (0.5, None, 1, 3, S1, False, None, True),
             (0.0, None, 2, 6, S2, False, BF, False)]


def test_sde_solver_across_calls(cuda_backend):
    ns = schedule()
    fn = sde_wrapper(ns)
    s = sde_solver(fn, ns)
    last = None
    for i, call in enumerate(SDE_CALLS):
        if call == "capture":
            # a graph of the previous call's configuration, with its generator registered: replay k is the eager run
            # of a fresh solver from the generator state just before it, and with eta > 0 the two replays differ
            eta, kind, order, steps, shape, cl, sd, thr = last
            gen, used = generator(kind, 100 + i)
            x = xs(i, shape, cl)
            kw = dict(steps=steps, order=order, eta=eta, generator=gen)
            g = s.capture(x, **kw)
            replays = []
            for k in range(2):
                st = used.get_state()
                replays.append(g(x).clone())
                after = used.get_offset()
                used.set_state(st)
                want = sde_solver(sde_wrapper(ns), ns, sd, thr).sample(x.clone(), **kw)
                assert same_bits(replays[-1], want) and used.get_offset() == after, (i, k)
            assert same_bits(replays[0], replays[1]) == (eta == 0), i
            del g
            continue
        last = call
        eta, kind, order, steps, shape, cl, sd, thr = call
        s.state_dtype = sd
        set_thresholding(s, thr)
        x = xs(i, shape, cl)
        kw = dict(steps=steps, order=order, eta=eta)
        gen, used = generator(kind, 100 + i)
        got = s.sample(x, generator=gen, **kw)
        off = used.get_offset()
        gen, used = generator(kind, 100 + i)
        want = sde_solver(sde_wrapper(ns), ns, sd, thr).sample(x.clone(), generator=gen, **kw)
        assert got.dtype == (sd or torch.float32) and same_bits(got, want), (i, call)
        assert off == used.get_offset(), (i, call)


@pytest.mark.parametrize("k", [2, 4])
def test_sde_run_stopped_by_the_network(cuda_backend, k):
    """The network raises at its k-th call: updates 1 .. k-1 have drawn their noise, so the generator sits where k-1
    draws of the contract leave it; the same solver then runs again as a fresh one does."""
    ns = schedule()
    plan = [k, 0]
    s = sde_solver(sde_wrapper(ns, make_net(raise_at=plan)), ns)
    x = xs(5)
    g = torch.Generator(DEV).manual_seed(31)
    with pytest.raises(Boom):
        s.sample(x, steps=6, order=2, eta=1.0, generator=g)
    g2 = torch.Generator(DEV).manual_seed(31)
    for _ in range(k - 1):
        torch.empty_like(x, dtype=torch.float32).normal_(generator=g2)
    assert g.get_offset() == g2.get_offset()
    plan[0] = 0                                  # (no more raising)
    got = s.sample(x, steps=6, order=2, eta=1.0, generator=torch.Generator(DEV).manual_seed(32))
    want = sde_solver(sde_wrapper(ns), ns).sample(x.clone(), steps=6, order=2, eta=1.0,
                                                   generator=torch.Generator(DEV).manual_seed(32))
    assert same_bits(got, want)


# ---- Perp-Neg --------------------------------------------------------------------------------------------------------

def perp_net(dtype):
    """test_perp_neg's network (conditional directions that differ nonlinearly; tame enough for the adaptive method),
    outputs in dtype[0] when set. Every run here is compared with another device run, so its transcendentals are
    fine."""
    from test_perp_neg import net

    def f(x, t, c):
        o = net(x, t, c)
        return o if dtype[0] is None else o.to(dtype[0])
    return f


def perp_wrapper(ns, K, scales, dtype):
    import dpm_solver_b200 as new
    return new.model_wrapper(perp_net(dtype), ns, model_type="noise", guidance_type="classifier-free",
                             condition=[torch.full((B, 1), float(k + 1), device=DEV) for k in range(K)],
                             unconditional_condition=torch.zeros(B, 1, device=DEV), guidance_scale=list(scales),
                             perp_neg=True)


SCALES = {2: [[7.5, -3.0], [4.0, 0.0], [1.0, -1.5]], 4: [[4.0, -1.0, -0.5, -2.5], [6.0, 0.0, -2.0, 1.0],
                                                        [3.0, -3.0, -3.0, -0.5]]}


@pytest.mark.parametrize("thr", [False, True])
def test_perp_neg_wrappers_across_calls(cuda_backend, thr):
    import dpm_solver_b200 as new
    ns = schedule()
    kw = dict(algorithm_type="dpmsolver++", correcting_x0_fn="dynamic_thresholding" if thr else None)
    dts = {2: [None], 4: [None]}
    fns = {K: perp_wrapper(ns, K, SCALES[K][0], dts[K]) for K in (2, 4)}
    solvers = {K: new.DPM_Solver(fns[K], ns, **kw) for K in (2, 4)}
    ad = dict(method="adaptive", order=2, atol=0.0078, rtol=0.05)
    # (K, scales index, x seed, shape, channels_last, output dtype, method)
    calls = [(2, 0, 1, S1, False, None, ad), (4, 0, 1, S1, False, None, ad),
             (2, 0, 1, S1, False, None, dict(steps=6, order=2)), (4, 1, 2, S2, True, None, dict(steps=5, order=3)),
             (2, 1, 2, S2, True, BF, dict(steps=6, order=2)), (4, 2, 3, S1, False, BF, dict(steps=6, order=2)),
             (2, 2, 3, S1, True, None, dict(steps=4, order=1)), (4, 0, 4, S2, False, None, dict(steps=6, order=2)),
             (2, 0, 1, S1, False, None, dict(steps=6, order=2))]
    for i, (K, si, seed, shape, cl, dt, skw) in enumerate(calls):
        scales = SCALES[K][si]
        fns[K].cond_scales = tuple(float(torch.tensor(v, dtype=torch.float32)) for v in scales)
        dts[K][0] = dt
        x = xs(seed, shape, cl)
        got = solvers[K].sample(x, **skw)
        want = new.DPM_Solver(perp_wrapper(ns, K, scales, [dt]), ns, **kw).sample(x.clone(), **skw)
        assert same_bits(got, want), (i, K, scales, shape, cl, dt)
