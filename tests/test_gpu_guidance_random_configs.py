"""CFG-Zero*, CFG++, regional guidance, TCFG, frequency-decoupled guidance and Perp-Neg in `sample()`, `UniPC.sample()`
and `inverse()` on the device over random configurations, bit for bit (tests/guidance_configs.py): paths A-E of
tests/test_gpu_apg_random_configs.py -- A the first call against the exact CPU executor (every intermediate and the
trace of network calls), B the same call again (no guided evaluation frozen as a `PreparedStep`, except FDG's, which is
one network output g: its frozen steps are served, and fall back when x comes in another layout), C another input on the
same solver against a fresh solver (the zero-init count starts over), D `capture()` replays (zero-init included; a mask
or an FDG [B, N] scale tensor read in place is rewritten after capture and the replay must follow it), E a fresh solver
on a second stream. A refused configuration raises on the device before any launch or network call. A module-wide tally
requires every path of interest to have been met by the fixed seeds."""
import pytest
import torch

from gpu_configs import DT, really_channels_last, same_bits
from guidance_configs import CHUNKS, PER_CHUNK, REQUIRED, REQUIRED_ON_DEVICE, SEED, GuidanceRig, configurations, \
    cpu_oracle, refused, tally_static
from oracle import ref_loader
from test_gpu_random_configs import LaunchSpy, distinct_ranges

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


def in_place_masks(rig, x):
    """Indices of the rig's masks that the launches read in place (contiguous fp32 on x's device in the map's layout)."""
    lay = "cl" if x.dim() == 4 and not x.is_contiguous() else "c"
    out = []
    for k, (m, cm) in enumerate(zip(rig.masks, rig.fn.cond_masks)):
        if m is not None and cm.weights(tuple(x.shape), lay, x.device)[0].data_ptr() == m.data_ptr():
            out.append(k)
    return out


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
        # device against device only (the error norm sums in another order than numpy), as for APG
        want = {"error": ValueError()} if refused(c) else None
    else:
        want = cpu_oracle(c)
    if want is not None and "error" in want:
        before = be.launch_count()
        rig = None
        with pytest.raises(ValueError):
            rig = GuidanceRig(new, c, "cuda:0")
            rig.sample(rig.solver(), rig.x(), trace=True)
        expect(be.launch_count() == before, "refused: the library launched")
        expect(not getattr(rig, "trace_log", None), "refused: the network was called")
        hit("rejected")
        return bad
    if want is not None and not torch.isfinite(want["y"].float()).all():
        hit("skipped:non-finite")
        return bad
    for k in tally_static(c):
        hit(k)
    if want is not None and "pinned" in want:
        hit("pinned")
    rig = GuidanceRig(new, c, "cuda:0")
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
        equal_runs(A, (want["y"], want["inter"]), "A vs CPU oracle")
    expect(same_bits(x, x_before), "A: x was modified")
    expect(distinct_ranges(A[1]), "A: intermediates overlap")
    keepA = [t.clone() for t in [A[0]] + A[1]]
    # ---- B: the same call again; no guided evaluation of these features is frozen ----
    before = be.launch_count()
    with LaunchSpy() as spy:
        Bv = rig.sample(s, x, trace=True)
    expect(be.launch_count() > before, "B: the library did not run")
    expect(Bv[2] == A[2], "B: trace of network calls")
    equal_runs(Bv, A, "B vs A")
    expect(all(same_bits(a, b) for a, b in zip([A[0]] + A[1], keepA)), "B overwrote a tensor run A returned")
    fdg = c["feature"] == "fdg"
    if unipc:
        expect(spy.dup + spy.plain + spy.fell_back == 0 and not s._prep_cache, "B: a UniPC run used a PreparedStep")
    elif fdg:
        # a frozen FDG step holds the one output g (a new allocation each evaluation: only its pointer is patched in)
        expect(all(k[5] and k[-1] for k in s._prep_cache), "B: an FDG step was frozen without g")
        if spy.dup + spy.plain and not bad:
            hit("fdg:frozen step served")
        if (s._prep_cache and x.is_contiguous() and len(c["shape"]) == 3
                and really_channels_last(dict(c, channels_last=True))):
            # the same solver on x in channels_last: g and the state in another layout than the frozen steps'
            xc = x.contiguous(memory_format=torch.channels_last)
            with LaunchSpy() as spy:
                Bc = rig.sample(s, xc, trace=True)
            fresh = GuidanceRig(new, c, "cuda:0")
            equal_runs(Bc, fresh.sample(fresh.solver(), xc.clone(), trace=True), "B: channels_last x vs fresh solver")
            expect(spy.fell_back > 0, "B: no frozen step fell back for a channels_last x")
            if spy.fell_back and not bad:
                hit("fdg:frozen step fell back")
    else:
        # (key field [5]: e_uncond is None -- a frozen step holds one network output, never a guided pair or a
        # Perp-Neg evaluation)
        expect(all(k[5] for k in s._prep_cache), "B: a guided step was frozen")
        if c["feature"] == "perp":
            expect(spy.dup + spy.plain == 0, "B: a Perp-Neg step was served by a PreparedStep")
    # ---- C: another input on the same solver against a fresh solver ----
    x2 = rig.x2()
    Cv = rig.sample(s, x2, trace=True)
    fresh = GuidanceRig(new, c, "cuda:0")
    Cw = fresh.sample(fresh.solver(), x2.clone(), trace=True)
    equal_runs(Cv, Cw, "C vs fresh solver")
    # (the adaptive method's number of evaluations follows its input: x2 may take other steps than x)
    expect(Cv[2] == Cw[2] and (adaptive or len(Cv[2]) == len(A[2])), "C: trace of network calls (the zero-init count)")
    # ---- D: graph capture and replay ----
    if not adaptive and not c["inverse"]:
        g = s.capture(x, **rig.kwargs())
        before = be.launch_count()
        expect(same_bits(g(x).clone(), A[0]), "D: replay of x vs A")
        expect(same_bits(g(x2).clone(), Cv[0]), "D: replay of x2 vs C")
        expect(same_bits(g(x).clone(), A[0]), "D: second replay of x vs A")
        expect(be.launch_count() == before, "D: a replay launched through the host path")
        equal_runs(rig.sample(s, x), A, "D: eager call after capture vs A")
        hit("captured")
        if c["zero_init"]:
            hit("captured:zero-init")
        if c["feature"] == "mask":
            ks = in_place_masks(rig, x)
            if ks:
                for k in ks:
                    rig.masks[k].mul_(-0.5).add_(0.75)
                got = g(x).clone()
                new_rig = GuidanceRig(new, c, "cuda:0", masks=[None if m is None else m.clone() for m in rig.masks])
                expect(same_bits(got, new_rig.sample(new_rig.solver(), x)[0]),
                       "D: replay after rewriting a mask vs a fresh eager run")
                hit("captured:rewritten-mask")
        if fdg and c["fdg_form"] == "rows":
            # an fp32 [B, N] tensor on the device is read in place: the replay follows a rewrite
            rig.fdg.mul_(-0.5).add_(0.75)
            got = g(x).clone()
            new_rig = GuidanceRig(new, c, "cuda:0", fdg=rig.fdg.clone())
            expect(same_bits(got, new_rig.sample(new_rig.solver(), x)[0]),
                   "D: replay after rewriting the FDG scales vs a fresh eager run")
            hit("captured:fdg rows rewritten")
        del g
    # ---- E: a fresh solver on a second stream ----
    side = torch.cuda.Stream()
    other = GuidanceRig(new, c, "cuda:0")
    s2 = other.solver()
    for _ in range(4):
        filler.mul_(1.0001)                              # ordinary work in flight on the default stream
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        Ev = other.sample(s2, x, trace=True)
    torch.cuda.current_stream().wait_stream(side)
    equal_runs(Ev, A, "E: second stream vs A")
    expect(Ev[2] == A[2], "E: trace of network calls")
    hit("second_stream")
    return bad


@pytest.mark.parametrize("chunk", range(CHUNKS))
def test_random_configurations_on_the_device(cuda_backend, chunk):
    filler = torch.ones(1 << 24, device="cuda:0")
    findings = []
    for i, c in enumerate(configurations(chunk)):
        try:
            bad = check_configuration(c, cuda_backend, filler)
        except Exception as e:          # reported with its configuration and seed, like a mismatch
            bad = ["%s: %s" % (type(e).__name__, str(e).splitlines()[0] if str(e) else "")]
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
