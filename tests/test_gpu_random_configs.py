"""`sample()` on the device over random configurations, bit for bit: the layer that strings the launches together
(prepared launches, the doubled CFG batch handed to the next network call, cached tables, graph capture, a second
stream) against the unmodified reference and the numpy executor run on CPU tensors (tests/gpu_configs.py).

Per configuration, ONE solver object on cuda:0 runs: A the first call (general path) against the CPU oracle, every
intermediate and the trace of network calls included; B the same call again (prepared launches) against A; C another
input against a fresh solver; D `capture()` replays against A and C, then an eager call; E a fresh solver on a second
stream against A. A module-wide tally requires every path of interest to have been met by the fixed seeds."""
import pytest
import torch

from gpu_configs import (CHUNKS, DT, PER_CHUNK, REQUIRED, REQUIRED_ON_DEVICE, SEED, Rig, configurations, cpu_oracle, freezable, rel_err,
                         same_bits, tally_static)
from oracle import ref_loader

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_loader.available(), reason="oracle/_ref not built and no reference tree")]
TALLY = {}
CHUNKS_RUN = set()
# max|y - y_ref| / max|y_ref| allowed where bit identity with the CPU executor does not hold end to end (see
# `tolerance`): the bound tests/test_gpu_cfg_rescale.py uses for fp32 state, and 16-bit storage precision
RESCALE_TOL, STORAGE_TOL = 1e-5, {"bf16": 2 ** -7, "f16": 2 ** -10}


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def tolerance(c):
    """None (bit identity with the CPU executor) or the relative bound of the one exempted family: the guidance
    rescale. Its per-sample ratio std(out_c)/std(g) is summed in fp32 by the device kernel and in fp64 by the
    executor, 2 ulp apart at most (test_gpu_cfg_rescale.py::test_ratio_kernel_vs_fp64), so a rescaled run agrees
    with the executor to rounding, not to the bit; with 16-bit state one such ulp can move a stored value by one
    16-bit step. Every other configuration -- 16-bit state with dynamic thresholding included, whose quantile and
    clamp read the same unrounded fp32 x0 in the kernels and in the executor -- is compared bit for bit."""
    if c["phi"] and (c["guidance"] != "rescale" or c["cfg"] != 1.0):
        return STORAGE_TOL[c["state_dtype"]] * 8 if c["state_dtype"] else RESCALE_TOL
    return None


def hit(key, n=1):
    TALLY[key] = TALLY.get(key, 0) + n


class LaunchSpy:
    """Counts `ops.PreparedStep.launch` calls by outcome while installed."""

    def __enter__(self):
        from dpm_solver_b200 import ops
        self.cls, self.orig = ops.PreparedStep, ops.PreparedStep.launch
        self.dup = self.plain = self.fell_back = 0
        spy = self

        def launch(prep, tensors):
            r = spy.orig(prep, tensors)
            if r is None:
                spy.fell_back += 1
            elif prep.dup:
                spy.dup += 1
            else:
                spy.plain += 1
            return r
        self.cls.launch = launch
        return self

    def __exit__(self, *exc):
        self.cls.launch = self.orig


def distinct_ranges(tensors):
    seen = {}
    for t in tensors:
        seen[id(t)] = (t.data_ptr(), t.data_ptr() + t.numel() * t.element_size())
    r = sorted(seen.values())
    return all(r[i][1] <= r[i + 1][0] for i in range(len(r) - 1))


def check_configuration(c, be, filler):
    """Runs A-E of one configuration; returns the list of findings (empty when everything agrees)."""
    import dpm_solver_b200 as new
    bad = []

    def expect(ok, what):
        if not ok:
            bad.append(what)

    def equal_runs(got, want, what):
        expect(same_bits(got[0], want[0]), what + ": y")
        expect(len(got[1]) == len(want[1]) and all(same_bits(a, b) for a, b in zip(got[1], want[1])),
               what + ": intermediates")

    adaptive = c["method"] == "adaptive"
    if adaptive:
        # device against device only: the error norm of the adaptive method sums in another order than torch and numpy
        # (tests/test_adaptive.py), so step sizes may differ in the last bits; only a refused construction is compared
        want = None
        try:
            Rig(new, c)
        except ValueError as e:
            want = {"error": e}
    else:
        want = cpu_oracle(c)
    if want is not None and "error" in want:
        with pytest.raises(type(want["error"])):
            rig = Rig(new, c, "cuda:0")
            rig.sample(rig.solver(), rig.x())
        hit("rejected")
        return bad
    if want is not None and not torch.isfinite(want["y"].float()).all():
        hit("skipped:non-finite")
        return bad
    for k in tally_static(c):
        hit(k)
    hit("reference" if want is not None and want.get("reference") else "executor only" if want else "device only")
    rig = Rig(new, c, "cuda:0")
    s = rig.solver()
    x = rig.x()
    x_before = x.clone()
    # ---- A: first call, general path ----
    A = rig.sample(s, x, trace=True)
    if adaptive and not torch.isfinite(A[0].float()).all():
        hit("skipped:non-finite")
        return bad
    expect(A[0].dtype == (DT[c["state_dtype"]] or torch.float32), "A: dtype")
    if want is not None:
        expect(A[2] == want["calls"], "A: trace of network calls")
        tol = tolerance(c)
        if tol is None:
            equal_runs(A, (want["y"], want["inter"]), "A vs CPU oracle")
        else:
            hit("tolerant")
            expect(len(A[1]) == len(want["inter"]), "A: number of intermediates")
            for i, (a, b) in enumerate(zip([A[0]] + A[1], [want["y"]] + want["inter"])):
                expect(a.dtype == b.dtype and rel_err(a, b) <= tol, "A vs CPU oracle within %g: tensor %d" % (tol, i))
    expect(same_bits(x, x_before), "A: x was modified")
    xs = x.untyped_storage().data_ptr()
    for i, t in enumerate(A[1]):
        # (the first intermediate of the multistep method is x_T itself, as in the reference, when no cast was needed)
        if not (t is x and i == 0 and c["method"] == "multistep"):
            expect(t.untyped_storage().data_ptr() != xs, "A: intermediate %d shares x's storage" % i)
    expect(A[0].untyped_storage().data_ptr() != xs, "A: y shares x's storage")
    expect(distinct_ranges(A[1]), "A: intermediates overlap")
    keepA = [t.clone() for t in [A[0]] + A[1]]
    # ---- B: the same call again, prepared launches ----
    before = be.launch_count()
    with LaunchSpy() as spy:
        Bv = rig.sample(s, x, trace=True)
    expect(be.launch_count() > before, "B: the library did not run")
    expect(Bv[2] == A[2], "B: trace of network calls")
    equal_runs(Bv, A, "B vs A")
    expect(distinct_ranges(Bv[1]), "B: intermediates overlap")
    expect(all(same_bits(a, b) for a, b in zip([A[0]] + A[1], keepA)), "B overwrote a tensor run A returned")
    if freezable(c):
        expect(len(s._prep_cache) > 0 and spy.dup + spy.plain > 0, "B: no prepared launch although one is eligible")
    hit("prepared:dup", spy.dup), hit("prepared:plain", spy.plain), hit("prepared:fell_back", spy.fell_back)
    hit("configurations with prepared launches", int(spy.dup + spy.plain > 0))
    # ---- C: another input on the same solver against a fresh solver ----
    x2 = rig.x2()
    with LaunchSpy() as spy:
        Cv = rig.sample(s, x2)
    hit("prepared:fell_back", spy.fell_back)
    hit("configurations that fell back", int(spy.fell_back > 0))
    fresh = Rig(new, c, "cuda:0")
    Cw = fresh.sample(fresh.solver(), x2.clone())
    equal_runs(Cv, Cw, "C vs fresh solver")
    # ---- D: graph capture and replay ----
    if not adaptive:
        kw = dict(steps=c["steps"], order=c["order"], skip_type=c["skip_type"], method=c["method"],
                  lower_order_final=c["lower_order_final"], denoise_to_zero=c["denoise_to_zero"],
                  solver_type=c["solver_type"], t_end=c["t_end"], t_start=c["t_start"])
        g = s.capture(x, **kw)
        before = be.launch_count()
        expect(same_bits(g(x).clone(), A[0]), "D: replay of x vs A")
        expect(same_bits(g(x2).clone(), Cv[0]), "D: replay of x2 vs C")
        expect(be.launch_count() == before, "D: a replay launched through the host path")
        equal_runs(rig.sample(s, x), A, "D: eager call after capture vs A")
        del g
        hit("captured")
    # ---- E: a fresh solver on a second stream (pinned asynchronous uploads, cached table views) ----
    side = torch.cuda.Stream()
    other = Rig(new, c, "cuda:0")
    s2 = other.solver()
    for _ in range(4):
        filler.mul_(1.0001)                              # ordinary work in flight on the default stream
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        Ev = other.sample(s2, x)
    torch.cuda.current_stream().wait_stream(side)
    equal_runs(Ev, A, "E: second stream vs A")
    equal_runs(other.sample(s2, x), A, "E: default stream after the second stream vs A")
    hit("second_stream")
    return bad


@pytest.mark.parametrize("chunk", range(CHUNKS))
def test_random_configurations_on_the_device(cuda_backend, chunk):
    filler = torch.ones(1 << 24, device="cuda:0")
    findings = []
    for i, c in enumerate(configurations(chunk)):
        cuda_backend.set_tuning(1 if c["tuning"] == "tma" else 2, 0, 0)
        try:
            bad = check_configuration(c, cuda_backend, filler)
        except Exception as e:          # reported with its configuration and seed, like a mismatch
            bad = ["%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")]
        finally:
            cuda_backend.set_tuning(2, 0, 0)
        if bad:
            findings.append((SEED + chunk, i, c, bad))
    CHUNKS_RUN.add(chunk)
    print("\nchunk %d: %d configurations, tally so far %s" % (chunk, PER_CHUNK, dict(sorted(TALLY.items()))))
    assert not findings, "\n".join("seed %d #%d %s\n    -> %s" % f for f in findings)


def test_tally_of_the_device_runs():
    """After the chunks: every path of interest was met (adjust the drawing weights, not this list)."""
    if len(CHUNKS_RUN) < CHUNKS:
        pytest.skip("needs all %d chunks of test_random_configurations_on_the_device in the same session" % CHUNKS)
    print("\ntally of %d configurations: %s" % (CHUNKS * PER_CHUNK, dict(sorted(TALLY.items()))))
    assert not [k for k in REQUIRED + REQUIRED_ON_DEVICE if not TALLY.get(k)]


# ---- what the random configurations found, reduced --------------------------------------------------------------
def test_capture_with_a_one_element_scale_tensor_on_the_device(cuda_backend):
    """A one-element `guidance_scale` tensor on the device is one scale, read on the host: once per (tensor, version),
    not at every evaluation -- a per-evaluation read synchronises and cannot be captured. (seed 9000 #0: B = 1 with
    per-sample scales.)"""
    import dpm_solver_b200 as new
    from test_gpu_solver_reuse import config
    for scales in ([3.5], [1.0]):
        rig = Rig(new, config(B=1, guidance="per_sample", scales=scales), "cuda:0")
        s, x = rig.solver(), rig.x()
        want = s.sample(x, steps=8, order=2)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            again = s.sample(x, steps=8, order=2)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert same_bits(again, want)
        g = s.capture(x, steps=8, order=2)
        assert same_bits(g(x).clone(), want)
        other = Rig(new, config(B=1, guidance="float", cfg=scales[0]), "cuda:0")
        assert same_bits(other.solver().sample(x, steps=8, order=2), want)
        rig.scale.fill_(7.5)                                  # a new value: read again, once
        other = Rig(new, config(B=1, guidance="float", cfg=7.5), "cuda:0")
        assert same_bits(s.sample(x, steps=8, order=2), other.solver().sample(x, steps=8, order=2))


@pytest.mark.parametrize("order", [2, 3])
def test_adaptive_device_controller_with_a_channels_last_network(cuda_backend, order):
    """The device controller commits accepted steps with a byte copy into its row-major state: a channels_last
    network's states are brought to that order first (seed 9000 #6 raised ValueError in select_copy). Same network
    calls and, to the reduction order of the error norm, the same sample as the host controller."""
    import dpm_solver_b200 as new
    from test_gpu_solver_reuse import call, config
    c = config(channels_last=True, guidance="float", cfg=3.5)
    kw = dict(method="adaptive", order=order, atol=0.05, rtol=0.2)
    rig = Rig(new, c, "cuda:0")
    y = call(rig.solver(), rig.x(), **kw)[0]
    plain = Rig(new, dict(c, channels_last=False), "cuda:0")
    assert same_bits(y, call(plain.solver(), plain.x(), **kw)[0])
    x_cl = plain.x().contiguous(memory_format=torch.channels_last)      # and a channels_last x_T (seed 9000 #3)
    assert same_bits(y, call(plain.solver(), x_cl, **kw)[0])
    host = rig.solver()
    host.adaptive_controller = "host"
    assert rel_err(y, call(host, rig.x(), **kw)[0]) <= 1e-3
