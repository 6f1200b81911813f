"""Cost of guidance rescale on the benchmark's CFG shapes.

    python tools/cfg_rescale_probe.py [--reps 50] [--samples 3]

For c3 (bf16 [2048,4,64,64], CFG 7.5, DPM-Solver-3 singlestep, 15 steps, eps) and c2 run with CFG 7.5
(bf16 [4096,4,64,64], DPM-Solver++2M, 20 steps) at phi = 0 and 0.7, prints one JSON line per case with
  - step_us:   one fused CFG step (singlestep difference form, both output copies), CUDA events over `reps` launches;
  - ratio_us / ratio_gbs / ratio_pct_peak: the ratio pass (2 launches) and its rate over 2*s_model bytes per element
               of x, against the H100 SXM data-sheet 3.35 TB/s;
  - sample_s:  end-to-end sample() with a synthetic network that returns pre-generated banks (bench.py's);
and the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {
    "c3": dict(shape=(2048, 4, 64, 64), algo="dpmsolver", method="singlestep", order=3, steps=15),
    "c2_cfg": dict(shape=(4096, 4, 64, 64), algo="dpmsolver++", method="multistep", order=2, steps=20),
}
PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def run(name, c, phi, reps, samples):
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper, ops
    from dpm_solver_b200._lib import FORM_DIFF2
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from cases import make_betas
    be = ops.backend()
    B, shape = c["shape"][0], c["shape"]
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
    banks = [torch.randn((2 * B,) + shape[1:], device="cuda", generator=g).to(torch.bfloat16) for _ in range(2)]
    banks[1][B:] = banks[1][B:] * 1.3 + 0.05
    out_u, out_c = banks[1].chunk(2)
    per_sample = x.numel() // B
    ratio = be.cfg_rescale_ratio(out_c, out_u, 7.5)
    x_in = torch.empty((2 * B,) + shape[1:], device="cuda", dtype=torch.bfloat16)
    a = ops.StepArgs(form=FORM_DIFF2, n_model=2, x=x, xe=x, m1=x, e_cond=out_c, e_uncond=out_u, guidance=7.5,
                     a=0.9, c0=-0.1, c1=0.2, w0=1.0, c0_on_old=True, state_dtype=torch.bfloat16,
                     out=x_in[:B], out2=x_in[B:])
    if phi:
        a.ratio, a.phi, a.per_sample = ratio, phi, per_sample
    step_us = timed(lambda: be.step(a), reps)
    ratio_us = timed(lambda: be.cfg_rescale_ratio(out_c, out_u, 7.5), reps) if phi else 0.0
    ratio_bytes = 2 * x.numel() * x.element_size()

    ns = NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    cnt = [0]

    def net(xx, tt, cc):
        cnt[0] += 1
        return banks[cnt[0] % 2]
    fn = model_wrapper(net, ns, guidance_type="classifier-free", condition=torch.ones(B, 1, device="cuda"),
                       unconditional_condition=torch.zeros(B, 1, device="cuda"), guidance_scale=7.5,
                       guidance_rescale=phi)
    s = DPM_Solver(fn, ns, algorithm_type=c["algo"], state_dtype=torch.bfloat16)
    kw = dict(steps=c["steps"], order=c["order"], method=c["method"])
    s.sample(x, **kw)
    times = []
    for _ in range(samples):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        s.sample(x, **kw)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    res = dict(case=name, phi=phi, step_us=round(step_us, 1), sample_s=round(min(times), 4),
               sample_s_all=[round(t, 4) for t in times], card=card())
    if phi:
        gbs = ratio_bytes / (ratio_us * 1e-6)
        res.update(ratio_us=round(ratio_us, 1), ratio_gbs=round(gbs / 1e9, 1), ratio_pct_peak=round(100 * gbs / PEAK, 1))
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--samples", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cfg_rescale_probe measures on the GPU; no CUDA device found")
    with torch.no_grad():
        for name, c in CASES.items():
            for phi in (0.0, 0.7):
                run(name, c, phi, args.reps, args.samples)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
