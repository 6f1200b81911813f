#!/usr/bin/env python
"""Small launches of every kernel family, meant to run under compute-sanitizer:

    compute-sanitizer --tool memcheck  python tools/sanitize_probe.py
    compute-sanitizer --tool racecheck python tools/sanitize_probe.py
    compute-sanitizer --tool synccheck python tools/sanitize_probe.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")):
    sys.path.insert(0, p)
import torch  # noqa: E402

from dpm_solver_b200 import ops  # noqa: E402
from dpm_solver_b200.ops import StepArgs  # noqa: E402

be = ops.CudaBackend()
dev = "cuda"
g = torch.Generator(device=dev).manual_seed(0)
mk = lambda n, dt=torch.float32: torch.randn(n, device=dev, generator=g).to(dt)
co = dict(a=0.95, c0=-0.1, c1=0.05, c2=-0.01, w0=1.02, w1=0.98, w2=0.51, w3=0.5, w4=0.33)
n = 8 * 148 * 1024 + 8 * 700 + 5          # > 1024 packets per SM: many tiles per SM on both variants, and a tail
for variant in (0, 1):
    be.set_tuning(variant, 0, 0)
    for dt in (torch.float32, torch.bfloat16):
        for form in (1, 3, 4, 5, 6):
            be.step(StepArgs(form=form, x=mk(n, dt), m0=mk(n, dt), m1=mk(n, dt), m2=mk(n, dt), **co))
        x = mk(n, dt)
        buf = torch.empty(2 * n + 8, device=dev, dtype=dt)
        be.step(StepArgs(form=5, n_model=2, x=x, xe=x, e_cond=mk(n, dt), e_uncond=mk(n, dt), m1=mk(n, dt), m2=mk(n, dt),
                         predict_x0=True, guidance=7.5, alpha_e=0.8, sigma_e=0.6, want_m_out=True, out=buf[:n], out2=buf[n:2 * n], **co))
        thr = torch.rand(5, device=dev) + 0.5
        nn = 5 * 8 * 2048
        be.step(StepArgs(form=4, n_model=1, x=mk(nn, dt), xe=mk(nn, dt), e_cond=mk(nn, dt), m1=mk(nn, dt), predict_x0=True,
                         alpha_e=0.8, sigma_e=0.6, thr=thr, per_sample=8 * 2048, want_m_out=True, **co))
be.set_tuning(2, 0, 0)
for per_sample, B in ((24, 7), (4 * 64 * 64, 5), (3 * 128 * 128, 3), (1001, 3)):
    for impl in ("pipeline", "cluster"):
        os.environ["DPM_QUANTILE_IMPL"] = impl
        a = StepArgs(form=0, n_model=2, xe=mk(per_sample * B), e_cond=mk(per_sample * B), e_uncond=mk(per_sample * B), predict_x0=True,
                     guidance=3.0, alpha_e=0.8, sigma_e=0.6, per_sample=per_sample, state_dtype=torch.float32)
        be.dynamic_threshold(a, 0.995, 1.0)
os.environ.pop("DPM_QUANTILE_IMPL", None)
be.error_norm(mk(4 * 3 * 1024).reshape(4, -1), mk(4 * 3 * 1024).reshape(4, -1), mk(4 * 3 * 1024).reshape(4, -1), 0.0078, 0.05)
# round 2: duplicate (TMA copy, two stores), reference-rounding vector kernels, in-kernel Philox noise, the
# device-side adaptive controller with launches that read their scalars from device memory
for dt in (torch.float32, torch.bfloat16):
    be.duplicate(mk(3 * 4 * 33 * 17, dt).reshape(3, 4, 33, 17))
    be.duplicate(mk(64 * 4 * 64 * 64, dt).reshape(64, 4, 64, 64))
nr = 8 * 5000 + 5
be.step(StepArgs(form=5, n_model=2, x=mk(nr), e_cond=mk(nr, torch.bfloat16), e_uncond=mk(nr, torch.bfloat16), m1=mk(nr), m2=mk(nr),
                 guidance=3.7, want_m_out=True, state_dtype=torch.float32, raw_round=1 | 4, **co))
be.add_noise_philox(mk(2 * 4 * 17 * 9).reshape(2, 4, 17, 9), [0.9, 0.5, 0.1], [0.43, 0.86, 0.99], torch.float32)
be.diffedit_corrector(mk(2 * 4 * 16 * 16).reshape(2, 4, 16, 16), mk(2 * 4 * 16 * 16).reshape(2, 4, 16, 16),
                      (mk(16 * 16).reshape(16, 16) > 0).float(), 0.8, 0.6)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from cases import exact_net, make_betas  # noqa: E402
from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper  # noqa: E402
import contextlib, io  # noqa: E402
for sched, algo in ((NoiseScheduleVP("linear"), "dpmsolver"), (NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1])), "dpmsolver++")):
    s = DPM_Solver(model_wrapper(exact_net, sched), sched, algorithm_type=algo)
    with contextlib.redirect_stdout(io.StringIO()):
        s.sample(mk(2 * 3 * 8 * 8).reshape(2, 3, 8, 8), method="adaptive", order=3, t_end=1e-3, solver_type="taylor")
torch.cuda.synchronize()
print("sanitize_probe: all kernel families launched")
