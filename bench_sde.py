"""Time one SDE-DPM-Solver++ 2M update at c2's shape against the ODE update and the unfused SDE update.

    python bench_sde.py [--iters 200] [--warmup 20]

Shape: bf16 state and network output, [4096, 4, 64, 64], DIFF2 (the 2M update), once with one network output and
once with classifier-free guidance. Three launches are timed with CUDA events over many warmed-up repetitions:
  (a) ode:     the fused ODE step (dpm_step)
  (b) sde:     the fused SDE step (dpm_step_sde): the same bytes, the noise drawn in registers
  (c) unfused: the ODE step, then torch's normal_ into an fp32 buffer, then x += cz*z (12 more bytes per element)
Prints one JSON line per case with the times, the algorithmic bytes and their share of 3.35 TB/s, and the card's name
and power limit read in the same run.
"""
import argparse
import json
import subprocess

import torch

from dpm_solver_b200 import ops
from dpm_solver_b200._lib import FORM_DIFF2

HBM = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) * 1e3 / iters      # us per launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    name, power = card()
    be = ops.backend()
    shape = (4096, 4, 64, 64)
    n = 4096 * 4 * 64 * 64
    bf = torch.bfloat16
    x, m1, ec, eu = (torch.randn(shape, device="cuda").to(bf) for _ in range(4))
    out, out2, m_out = (torch.empty(shape, device="cuda", dtype=bf) for _ in range(3))
    z = torch.empty(shape, device="cuda", dtype=torch.float32)
    g = torch.Generator("cuda").manual_seed(0)
    cz = 0.3
    for ne in (1, 2):
        args = ops.StepArgs(form=FORM_DIFF2, n_model=ne, x=x, xe=x, m1=m1, e_cond=ec, e_uncond=eu if ne == 2 else None,
                            predict_x0=True, alpha_e=0.8, sigma_e=0.6, guidance=7.5, a=0.9, c0=0.1, c1=-0.2, w0=1.1,
                            want_m_out=True, out=out, m_out=m_out, out2=out2 if ne == 2 else None)
        sde = ops.StepArgs(**{f: getattr(args, f) for f in args.__dataclass_fields__})
        sde.sde = ops.SdeNoise(cz, g)

        def unfused():
            be.step(args)
            z.normal_(generator=g)
            out.add_(z, alpha=cz)

        t_ode = timed(lambda: be.step(args), a.iters, a.warmup)
        t_sde = timed(lambda: be.step(sde), a.iters, a.warmup)
        t_unf = timed(unfused, a.iters, a.warmup)
        # bytes per element: read x, e_c [, e_u], m1; write out [, out2], m_out
        bpe = 2 * (5 if ne == 1 else 7)
        res = {"case": "c2_bf16_2m_sde" + ("_cfg" if ne == 2 else ""), "shape": list(shape),
               "us_ode": round(t_ode, 1), "us_sde": round(t_sde, 1), "us_unfused": round(t_unf, 1),
               "sde_over_ode": round(t_sde / t_ode, 3), "sde_speedup_vs_unfused": round(t_unf / t_sde, 3),
               "bytes_per_elem": bpe, "unfused_bytes_per_elem": bpe + 12,
               "tbs_ode": round(bpe * n / t_ode / 1e6, 3), "tbs_sde": round(bpe * n / t_sde / 1e6, 3),
               "hbm_share_sde": round(bpe * n / (t_sde * 1e-6) / HBM, 3), "gpu": name, "power_limit": power}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
