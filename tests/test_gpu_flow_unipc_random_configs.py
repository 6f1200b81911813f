"""Flow-matching and UniPC `sample()` on the device over random configurations, bit for bit (tests/flow_unipc_configs.py):
paths A-E of tests/test_gpu_random_configs.py -- A the first call against the CPU oracle (every intermediate and the
trace of network calls), B the same call again, C another input against a fresh solver, D `capture()` replays, E a fresh
solver on a second stream -- with the sampler's own arguments. UniPC launches are never frozen: its B runs no
`PreparedStep`. A refused configuration raises the executor's exception on the device and launches nothing. A
module-wide tally requires every path of interest to have been met by the fixed seeds."""
import pytest
import torch

from flow_unipc_configs import (CHUNKS, PER_CHUNK, REQUIRED, REQUIRED_ON_DEVICE, SEED, FlowRig, configurations, cpu_oracle,
                                tally_static)
from gpu_configs import DT, freezable, rel_err, same_bits
from oracle import ref_loader
from test_gpu_random_configs import LaunchSpy, distinct_ranges, tolerance

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_loader.available(), reason="oracle/_ref not built and no reference tree")]
TALLY = {}
CHUNKS_RUN = set()


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def hit(key, n=1):
    TALLY[key] = TALLY.get(key, 0) + n


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

    unipc = c["sampler"] == "unipc"
    adaptive = not unipc and c["method"] == "adaptive"
    if adaptive:
        # device against device only (the error norm sums in another order than numpy); a refusal is compared
        want = None
        try:
            FlowRig(new, c).solver()
        except ValueError as e:
            want = {"error": e}
    else:
        want = cpu_oracle(c)
    if want is not None and "error" in want:
        before = be.launch_count()
        with pytest.raises(type(want["error"])):
            rig = FlowRig(new, c, "cuda:0")
            rig.sample(rig.solver(), rig.x())
        expect(be.launch_count() == before, "refused: the library launched")
        hit("rejected")
        return bad
    if want is not None and not torch.isfinite(want["y"].float()).all():
        hit("skipped:non-finite")
        return bad
    for k in tally_static(c):
        hit(k)
    hit("pinned:" + want["pinned"] if want is not None and "pinned" in want else
        "executor only" if want is not None else "device only")
    rig = FlowRig(new, c, "cuda:0")
    s = rig.solver()
    x = rig.x()
    x_before = x.clone()
    # ---- A: first call ----
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
        # (the first intermediate is x_T itself when no cast was needed)
        if not (t is x and i == 0 and (unipc or c["method"] == "multistep")):
            expect(t.untyped_storage().data_ptr() != xs, "A: intermediate %d shares x's storage" % i)
    expect(A[0].untyped_storage().data_ptr() != xs, "A: y shares x's storage")
    expect(distinct_ranges(A[1]), "A: intermediates overlap")
    keepA = [t.clone() for t in [A[0]] + A[1]]
    # ---- B: the same call again: prepared launches for DPM_Solver, none for UniPC ----
    before = be.launch_count()
    with LaunchSpy() as spy:
        Bv = rig.sample(s, x, trace=True)
    expect(be.launch_count() > before, "B: the library did not run")
    expect(Bv[2] == A[2], "B: trace of network calls")
    equal_runs(Bv, A, "B vs A")
    expect(distinct_ranges(Bv[1]), "B: intermediates overlap")
    expect(all(same_bits(a, b) for a, b in zip([A[0]] + A[1], keepA)), "B overwrote a tensor run A returned")
    if unipc:
        expect(spy.dup + spy.plain + spy.fell_back == 0 and not s._prep_cache, "B: a UniPC run used a PreparedStep")
    elif freezable(c):
        expect(len(s._prep_cache) > 0 and spy.dup + spy.plain > 0, "B: no prepared launch although one is eligible")
    hit("prepared", int(spy.dup + spy.plain > 0))
    # ---- C: another input on the same solver against a fresh solver ----
    x2 = rig.x2()
    Cv = rig.sample(s, x2)
    fresh = FlowRig(new, c, "cuda:0")
    Cw = fresh.sample(fresh.solver(), x2.clone())
    equal_runs(Cv, Cw, "C vs fresh solver")
    # ---- D: graph capture and replay ----
    if not adaptive:
        g = s.capture(x, **rig.kwargs())
        before = be.launch_count()
        expect(same_bits(g(x).clone(), A[0]), "D: replay of x vs A")
        expect(same_bits(g(x2).clone(), Cv[0]), "D: replay of x2 vs C")
        expect(be.launch_count() == before, "D: a replay launched through the host path")
        equal_runs(rig.sample(s, x), A, "D: eager call after capture vs A")
        del g
        hit("captured")
    # ---- E: a fresh solver on a second stream ----
    side = torch.cuda.Stream()
    other = FlowRig(new, c, "cuda:0")
    s2 = other.solver()
    for _ in range(4):
        filler.mul_(1.0001)                              # ordinary work in flight on the default stream
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        Ev = other.sample(s2, x, trace=True)
    torch.cuda.current_stream().wait_stream(side)
    equal_runs(Ev, A, "E: second stream vs A")
    expect(Ev[2] == A[2], "E: trace of network calls")
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
