"""SDE-DPM-Solver++ `sample()` on the device over random configurations (tests/sde_configs.py), bit for bit against the
executor drawing from the same CUDA generator. Per configuration, from a re-seeded generator before every run that
draws: A the first call against `sde_configs.oracle` on the device (y, every intermediate, the trace of network calls,
the generator's final offset); B the same call again (the same bits; with eta > 0 no step is frozen, with eta = 0 the
frozen steps are served and the run is still the "dpmsolver++" run); C another input on the same solver against a
fresh solver; D `capture()` with the generator registered (replay k is the eager run from the generator state just
before it -- the torch-drawn, read-from-memory noise against the in-kernel draw -- and two replays differ when
eta > 0); E a fresh solver on a second stream. A refused configuration raises and launches nothing. A module-wide
tally requires every path of interest to have been met by the fixed seeds."""
import traceback

import pytest
import torch

from gpu_configs import DT, rel_err, same_bits
from sde_configs import CHUNKS, PER_CHUNK, REQUIRED, REQUIRED_ON_DEVICE, SEED, SdeRig, _ode_run, configurations, \
    default_generator, oracle, refused, tally_static
from test_gpu_random_configs import LaunchSpy, distinct_ranges

pytestmark = pytest.mark.gpu
TALLY = {}
CHUNKS_RUN = set()
DEV = "cuda:0"
# the guidance rescale's per-sample ratio is summed in fp32 on the device and in fp64 by the executor
# (tests/test_gpu_random_configs.py::tolerance): a rescaled run agrees to rounding, every other one to the bit
RESCALE_TOL, STORAGE_TOL = 1e-5, {"bf16": 2 ** -7, "f16": 2 ** -10}


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def hit(key, n=1):
    TALLY[key] = TALLY.get(key, 0) + n


def tolerance(c):
    if c["phi"] and c["cfg"] != 1.0:
        return STORAGE_TOL[c["state_dtype"]] * 8 if c["state_dtype"] else RESCALE_TOL
    return None


def check_configuration(c, be, filler):
    """Runs A-E of one configuration; returns the list of findings (empty when everything agrees)."""
    import dpm_solver_b200 as new
    bad = []
    seed = c["seed"]
    tol = tolerance(c)

    def expect(ok, what):
        if not ok:
            bad.append(what)

    def equal_runs(got, want, what, tol=None):
        if tol is None:
            expect(same_bits(got[0], want[0]), what + ": y")
        else:
            expect(rel_err(got[0], want[0]) <= tol, what + ": y (%g)" % rel_err(got[0], want[0]))
        expect(len(got[1]) == len(want[1]) and all(same_bits(a, b) if tol is None else rel_err(a, b) <= tol
                                                   for a, b in zip(got[1], want[1])), what + ": intermediates")

    if refused(c):
        before = be.launch_count()
        rig = used = None
        with pytest.raises(ValueError):
            rig = SdeRig(new, c, DEV)
            s = rig.solver()
            gen = rig.generator(seed)
            used = gen if isinstance(gen, torch.Generator) else default_generator(DEV)
            state = used.get_state()
            rig.sample(s, rig.x(), trace=True, gen=gen)
        expect(be.launch_count() == before, "refused: the library launched")
        expect(not getattr(rig, "trace_log", None), "refused: the network was called")
        expect(used is None or torch.equal(used.get_state(), state), "refused: the generator moved")
        hit("rejected")
        return bad
    want = oracle(c, DEV, seed)
    assert "error" not in want, want
    if not torch.isfinite(want["y"].float()).all():
        hit("skipped:non-finite")
        return bad
    for k in tally_static(c):
        hit(k)
    rig = SdeRig(new, c, DEV)
    s = rig.solver()
    x = rig.x()
    x_before = x.clone()

    def run(solver, xx, fresh_rig=None, **kw):
        r = fresh_rig or rig
        gen = r.generator(seed)
        used = gen if gen is not None else default_generator(DEV)
        out = r.sample(solver, xx, trace=True, gen=gen, **kw)
        return out, used.get_offset()

    # ---- A: first call ----
    A, offA = run(s, x)
    if want["offset"] is None:
        want["offset"] = 0                       # (eta = 0 draws nothing: the offset stays where seeding put it)
    expect(A[0].dtype == (DT[c["state_dtype"]] or torch.float32), "A: dtype")
    expect(A[2] == want["calls"], "A: trace of network calls")
    equal_runs(A, (want["y"], want["inter"]), "A vs the executor", tol)
    expect(offA == want["offset"], "A: generator offset %d vs %d" % (offA, want["offset"]))
    expect(same_bits(x, x_before), "A: x was modified")
    expect(distinct_ranges(A[1]), "A: intermediates overlap")
    # ---- B: the same call again, from the same generator state ----
    n_prep = len(s._prep_cache)
    with LaunchSpy() as spy:
        (Bv, offB) = run(s, x)
    expect(Bv[2] == A[2] and offB == offA, "B: trace of network calls / generator offset")
    equal_runs(Bv, A, "B vs A")
    if c["eta"]:
        expect(len(s._prep_cache) == n_prep and spy.dup + spy.plain + spy.fell_back == 0,
               "B: a step with noise was frozen")
    else:
        if spy.dup + spy.plain:
            hit("frozen eta=0 step served")
        ode = SdeRig(new, dict(c, algo="dpmsolver++"), DEV)
        equal_runs(Bv, _ode_run(ode), "B: eta=0 vs the dpmsolver++ run")
    # ---- C: another input on the same solver against a fresh solver ----
    x2 = rig.x2()
    Cv, offC = run(s, x2)
    fresh = SdeRig(new, c, DEV)
    Cw, offCw = run(fresh.solver(), x2.clone(), fresh)
    equal_runs(Cv, Cw, "C vs fresh solver")
    expect(Cv[2] == Cw[2] and offC == offCw, "C: trace of network calls / generator offset")
    # ---- D: capture with the generator registered ----
    gen = rig.generator(seed)
    used = gen if gen is not None else default_generator(DEV)
    kw = dict(rig.kwargs(), eta=c["eta"], generator=gen)
    g = s.capture(x, **kw)
    st0 = used.get_state()
    r1 = g(x).clone()
    st1 = used.get_state()
    r2 = g(x).clone()
    expect(same_bits(r1, r2) == (c["eta"] == 0), "D: two replays %s" % ("differ" if c["eta"] == 0 else "agree"))
    for st, r in ((st0, r1), (st1, r2)):
        used.set_state(st)
        expect(same_bits(r, s.sample(x, **kw)), "D: replay vs the eager run from its generator state")
    del g
    hit("captured")
    if c["eta"]:
        hit("captured:eta>0")
    # ---- E: a fresh solver on a second stream ----
    side = torch.cuda.Stream()
    other = SdeRig(new, c, DEV)
    s2 = other.solver()
    for _ in range(4):
        filler.mul_(1.0001)                              # ordinary work in flight on the default stream
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        Ev, offE = run(s2, x, other)
    torch.cuda.current_stream().wait_stream(side)
    equal_runs(Ev, A, "E: second stream vs A")
    expect(Ev[2] == A[2] and offE == offA, "E: trace of network calls / generator offset")
    hit("second_stream")
    return bad


@pytest.mark.parametrize("chunk", range(CHUNKS))
def test_random_configurations_on_the_device(cuda_backend, chunk):
    filler = torch.ones(1 << 24, device=DEV)
    findings = []
    for i, c in enumerate(configurations(chunk)):
        try:
            bad = check_configuration(c, cuda_backend, filler)
        except Exception as e:          # reported with its configuration and seed, like a mismatch
            where = traceback.extract_tb(e.__traceback__)[-1]
            bad = ["%s: %s (%s:%d)" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "",
                                       where.filename.split("/")[-1], where.lineno)]
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


def test_correcting_xt_fn_draws_in_program_order(cuda_backend):
    """A correcting_xt_fn that draws from the run's CUDA generator sees the values the contract's program order gives:
    its own draws interleaved with each update's empty_like(x, dtype=float32).normal_."""
    import dpm_solver_b200 as new
    ns = new.NoiseScheduleVP("discrete", betas=torch.linspace(1e-4, 2e-2, 1000))
    g = torch.Generator(DEV).manual_seed(9)
    x = torch.randn(3, 4, 16, 16, generator=torch.Generator(DEV).manual_seed(1), device=DEV)
    hook = []

    def xt_fn(xt, t, step):
        hook.append(torch.randn(5, generator=g, device=DEV))
        return xt

    fn = new.model_wrapper(lambda xx, tt: 0.3 * xx + 0.1, ns, model_type="noise")
    new.DPM_Solver(fn, ns, algorithm_type="sde-dpmsolver++", correcting_xt_fn=xt_fn).sample(
        x, steps=5, order=2, eta=1.0, generator=g)
    g2 = torch.Generator(DEV).manual_seed(9)
    expect = [torch.randn(5, generator=g2, device=DEV)]      # (the hook also runs at the initial state)
    for _ in range(5):
        torch.empty_like(x, dtype=torch.float32).normal_(generator=g2)
        expect.append(torch.randn(5, generator=g2, device=DEV))
    assert g.get_offset() == g2.get_offset()
    assert len(hook) == len(expect) and all(torch.equal(a, b) for a, b in zip(hook, expect))
