"""The SDE and UniPC step kernels at IEEE edges, on every dispatch path, against the numpy executors.

Cases come from tests/sde_unipc_edges.py: NaN, +-inf, -0 and subnormal operands (tests/step_edges.py), x0 numerators at
the range guard of the constant division, clamp numerators at GUARD_TINY under accepted thresholds, thresholds that
are 0, +-inf, NaN, subnormal or refused, alpha_e on both sides of recip_div_ok, per-sample scales, ratios, CFG-Zero* s*
and TCFG words from {0, -0, 1, NaN, +-inf, subnormal, ordinary}, cz in {0, -0, 1e-40, 3e38, 0.37} and fp16 results on
both sides of 65520 (o + cz*z for SDE; the corrected state and the predictor output for UniPC). Each runs on the
device and in the executor (SdeOracle with the launch's own z, drawn beforehand from a copy of its generator; the
UniPC executor): m_out, out, out2 and out_c must be bit-identical with NaN in the same places, and the generator must
advance as normal_ advances it.

The dispatch mirror names the kernel and path of every launch (FAST or generic instantiation, guidance kind, packet or
element path per noise segment, the UniPC body and its scalar tail); the test tallies (family, kernel, path, division
site, recip / ieee) and requires the rare ones. torch.profiler confirms the mirror on one launch per kernel kind.
The single-rounding pin plants lanes of 16-bit SDE launches where rounding the update before adding cz*z would give
other bits. A bf16 launch just above 2^29 elements checks the second noise segment's unaligned base."""
import os
import subprocess
import sys
from collections import Counter

import numpy as np
import pytest
import torch

from dpm_solver_b200._lib import FORM_DIFF2, PARAM_NOISE
from dpm_solver_b200.ops import SdeNoise, StepArgs
from edm_oracle import EDMOracle
from sde_unipc_edges import (BF16, F32, GivenNoise, build_sde, build_unipc, guard_hits, kernel_name, noise_segments,
                             plant_noise, planted_hits, required, required_hits, sde_paths, sde_specs, tally_launch,
                             to_device, unipc_mirror, unipc_specs)
from step_edges import assert_bits_equal, recip_div_ok

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(autouse=True)
def peak_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    assert torch.cuda.max_memory_allocated() <= 12 * 2 ** 30


def _gen(seed):
    return torch.Generator("cuda").manual_seed(seed)


def _fp64_check(tally, a, m):
    """fp32 noise launches without thresholds or per-sample words: m_out = fl32(float64(num) / float64(alpha))."""
    if m is None or a.state_dtype != F32 or a.e_cond.dtype != F32 or not a.predict_x0 or a.param != PARAM_NOISE \
            or a.thr is not None or any(getattr(a, f, None) is not None
                                        for f in ("ratio", "guidance_b", "cfgzero_s", "tcfg_w")):
        return
    with np.errstate(all="ignore"):
        eps = a.e_cond.numpy().reshape(-1)
        if a.n_model == 2:
            epu = a.e_uncond.numpy().reshape(-1)
            eps = epu + f32(a.guidance) * (eps - epu)
        num = a.xe.numpy().reshape(-1) - f32(a.sigma_e) * eps
        want = (num.astype(np.float64) / np.float64(f32(a.alpha_e))).astype(f32)
    got = m.cpu().numpy().reshape(-1)
    fin = np.isfinite(got)
    assert (got[fin].view(np.uint32) == want[fin].view(np.uint32)).all(), "fp64 quotient"
    tally[("fp64 checked", "recip" if recip_div_ok(f32(a.alpha_e)) else "ieee")] += int(fin.sum())


def run_sde(be, spec, tally=None, hits=None):
    a, info = build_sde(spec)
    g = _gen(spec["seed"])
    clone = _gen(spec["seed"])
    clone.set_offset(g.get_offset())
    z = torch.empty(info["n"], device="cuda").normal_(generator=clone).cpu()
    plant_noise(a, info, z.numpy())
    d = to_device(a, spec["path"])
    d.sde = SdeNoise(a.sde.cz, g)
    gm, go = be.step(d)
    with np.errstate(all="ignore"):
        wm, wo = GivenNoise(z).step(a)
    what = "%s %s" % (spec, dict(param=a.param, px0=a.predict_x0, alpha=a.alpha_e, cz=a.sde.cz,
                                 thr=None if a.thr is None else a.thr.tolist()))
    assert g.get_offset() == clone.get_offset(), what
    for got, want, name in ((gm, wm, "m_out"), (go, wo, "out"), (d.out2, a.out2, "out2")):
        assert (got is None) == (want is None), (name, what)
        if got is not None:
            assert_bits_equal(got, want, "%s of %s" % (name, what))
    if tally is not None:
        runs = tally_launch(tally, spec, a, info)
        guard_hits(hits, spec, a, info, runs)
        planted_hits(hits, spec, info)
        _fp64_check(tally, a, gm)
    kern, segs = sde_paths(a, spec["md"], info["n"], spec["path"] != "unaligned", spec["path"] == "zgiven")
    return [kern] * len(segs)


def run_unipc(be, spec, tally=None, hits=None):
    a, info = build_unipc(spec)
    d = to_device(a, spec["path"])
    gm, go = be.step(d)
    with np.errstate(all="ignore"):
        wm, wo = EDMOracle().step(a)
    what = "%s %s" % (spec, dict(param=a.param, px0=a.predict_x0, alpha=a.alpha_e, words=a.unipc,
                                 thr=None if a.thr is None else a.thr.tolist()))
    for got, want, name in ((gm, wm, "m_out"), (go, wo, "out"), (d.out2, a.out2, "out2"), (d.out_c, a.out_c, "out_c")):
        assert (got is None) == (want is None), (name, what)
        if got is not None:
            assert_bits_equal(got, want, "%s of %s" % (name, what))
    if tally is not None:
        guard_hits(hits, spec, a, info, tally_launch(tally, spec, a, info))
        planted_hits(hits, spec, info)
        _fp64_check(tally, a, gm)
    return unipc_mirror(a, spec["md"], info["n"], spec["path"] != "unaligned")


REQUIRED_FP64 = [("fp64 checked", "recip"), ("fp64 checked", "ieee")]


def test_sde_and_unipc_kernels_at_ieee_edges(cuda_backend):
    tally, hits = Counter(), Counter()
    sde, uni = sde_specs(), unipc_specs()
    for spec in sde:
        run_sde(cuda_backend, spec, tally, hits)
    for spec in uni:
        run_unipc(cuda_backend, spec, tally, hits)
    print("\n%d SDE and %d UniPC edge-valued launches; path tally:" % (len(sde), len(uni)))
    for k, v in sorted(tally.items(), key=str):
        print("  %-70s %d" % (k, v))
    print("numerator, boundary and pin hits:", dict(sorted(hits.items(), key=str)))
    missing = [k for k in required() + REQUIRED_FP64 if tally[k] == 0] + [k for k in required_hits() if hits[k] == 0]
    assert not missing, missing


def profile_mirror():
    """The dispatch mirror against torch.profiler's kernel names, one launch per kind of kernel, one profiler session
    each."""
    from dpm_solver_b200 import ops
    from torch.profiler import ProfilerActivity, profile
    be = ops.CudaBackend()
    chosen = {}
    for spec in sde_specs():
        a, info = build_sde(spec)
        kern, segs = sde_paths(a, spec["md"], info["n"], spec["path"] != "unaligned", spec["path"] == "zgiven")
        key = ("sde", kern[3], kern[5], kern[6], kern[1] == kern[2] == F32 and kern[3] == 0 and spec["ne"] > 0,
               segs[0][2] > 0, segs[0][3] > 0)
        chosen.setdefault(key, (run_sde, spec))
    for spec in unipc_specs():
        a, info = build_unipc(spec)
        ks = unipc_mirror(a, spec["md"], info["n"], spec["path"] != "unaligned")
        key = ("unipc", ks[0][3:] if ks[0][0] == "unipc" else (), len(ks))
        chosen.setdefault(key, (run_unipc, spec))
    assert len(chosen) >= 20, chosen.keys()
    for run, spec in chosen.values():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ks = run(be, spec)
            torch.cuda.synchronize()
        ran = [e.name.replace(" ", "") for e in prof.events() if "k_step_" in e.name]
        want = [kernel_name(k) for k in ks]
        assert len(ran) == len(want) and all(w in r for w, r in zip(want, ran)), (spec, want, ran)
    print("%d profiled launches match the mirror" % len(chosen))


def test_mirror_names_the_kernel_that_ran():
    """profile_mirror() in a child process of its own, like the profiler check of tests/test_gpu_step_edges.py."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path[:0] = %r; import test_gpu_sde_unipc_edges as t; t.profile_mirror()"
            % [root, os.path.join(root, "tests"), os.path.join(root, "tests", "golden")])
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=root, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-4000:], r.stderr[-4000:])
    print(r.stdout.strip().splitlines()[-1])


def test_full_size_launch_with_an_unaligned_second_segment(cuda_backend):
    """A bf16 DIFF2 launch of 3 samples of 178956984 elements (2^29 + 40 in all) with a model stage and per-sample
    thresholds: its draw is split into two segments, the second based at element 268435476 (not a multiple of 8), so
    that segment takes the element path with per-sample reads. Slices at the start, across the seam and at the end
    equal the executor's on the same noise."""
    B, ps = 3, 178956984
    n = B * ps
    segs = noise_segments(n)
    assert len(segs) == 2 and segs[1][0] % 8 == 4 and ps % 8 == 0
    g = _gen(21)
    x, m1, ec = (torch.randn(n, device="cuda", generator=g).to(BF16) for _ in range(3))
    thr = torch.tensor([1.3, 0.6, 2.5], device="cuda")
    kw = dict(form=FORM_DIFF2, n_model=1, param=PARAM_NOISE, predict_x0=True, alpha_e=0.8, sigma_e=0.6, a=0.9, c0=0.1,
              c1=-0.2, w0=1.1, want_m_out=True, state_dtype=BF16)
    a = StepArgs(x=x, xe=x, m1=m1, e_cond=ec, thr=thr, per_sample=ps, sde=SdeNoise(0.37, g), **kw)
    kern, paths = sde_paths(a, BF16, n, True, False)
    assert paths[0][2] > 0 and paths[1][2] == 0 and paths[1][3] == paths[1][1], paths
    clone = _gen(21)
    clone.set_offset(g.get_offset())
    m, out = cuda_backend.step(a)
    del a
    z = torch.empty(n, device="cuda").normal_(generator=clone)
    assert g.get_offset() == clone.get_offset()
    L, seam = 4096, segs[1][0]
    for s0 in (0, seam - L // 2 - 3, n - L):
        sl = slice(s0, s0 + L)
        b = s0 // ps
        assert (s0 + L - 1) // ps == b
        h = StepArgs(x=x[sl].cpu(), xe=None, m1=m1[sl].cpu(), e_cond=ec[sl].cpu(), thr=thr[b:b + 1].cpu(),
                     per_sample=L, sde=SdeNoise(0.37), **kw)
        h.xe = h.x
        with np.errstate(all="ignore"):
            wm, wo = GivenNoise(z[sl].cpu()).step(h)
        assert_bits_equal(out[sl], wo, "out at %d" % s0)
        assert_bits_equal(m[sl], wm, "m_out at %d" % s0)
