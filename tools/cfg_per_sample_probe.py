"""Cost of per-sample classifier-free guidance scales at the c3 shape.

    python tools/cfg_per_sample_probe.py [--reps 30] [--rounds 5] [--samples 10]

c3: bf16 [2048,4,64,64], CFG, DPM-Solver-3 singlestep, 15 steps. Prints one JSON line per case:
  - step_*: one fused step with one scale (7.5) and with a per-sample scale tensor, on the same network outputs. Each
    round times `reps` launches with CUDA events (per-launch median); the two are alternated over `rounds` rounds and the
    median of the rounds is reported. Cases: the c3 DIFF2 step (bf16, noise network, vector FAST kernels); an fp32-state
    v-network DIFF2 step predicting x0 (the generic vector kernels); an fp32-state SS3T step (FAST).
  - sample_*: end-to-end sample() with a synthetic network that returns pre-generated banks (bench.py's), one scale vs
    four mixed scales, `samples` alternated runs: device time (CUDA events around the call) and host time until the
    call returns (the enqueue cost), medians in µs. Cases: c3; and a v network with dynamic thresholding, where the
    guided noise is materialised in fp32 and the step then runs on the element-wise kernel.
The card's name, PCI bus id, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPE = (2048, 4, 64, 64)


def card():
    """Name, power limit and SM clock of the card this process runs on, queried by its PCI bus id (torch's device
    index is not nvidia-smi's under CUDA_VISIBLE_DEVICES)."""
    pr = torch.cuda.get_device_properties(torch.cuda.current_device())
    bus = "%08X:%02X:%02X.0" % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
    q = subprocess.run(["nvidia-smi", "--id=" + bus, "--query-gpu=name,pci.bus_id,power.limit,clocks.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def launch_median_us(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) * 1e3 for a, b in ev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--samples", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cfg_per_sample_probe measures on the GPU; no CUDA device found")
    import dataclasses
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, model_wrapper, ops
    from dpm_solver_b200._lib import FORM_DIFF2, FORM_SS3T, PARAM_V
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from cases import make_betas
    torch.set_grad_enabled(False)
    be = ops.backend()
    B = SHAPE[0]
    g = torch.Generator(device="cuda").manual_seed(0)
    vals = [7.5, 3.0, 12.0, 1.0]
    scales = torch.tensor([vals[b % 4] for b in range(B)], dtype=torch.float32, device="cuda")
    rnd = lambda shape, dt: torch.randn(shape, device="cuda", generator=g).to(dt)
    bf = torch.bfloat16
    x = rnd(SHAPE, bf)
    banks = [rnd((2 * B,) + SHAPE[1:], bf) for _ in range(2)]
    card_s = card()

    def step_case(name, a):
        ag = dataclasses.replace(a, guidance_b=scales, per_sample=a.e_cond.numel() // B)
        be.step(a), be.step(ag)
        one, per = [], []
        for _ in range(args.rounds):
            one.append(launch_median_us(lambda: be.step(a), args.reps))
            per.append(launch_median_us(lambda: be.step(ag), args.reps))
        so, sp = statistics.median(one), statistics.median(per)
        print(json.dumps(dict(case=name, step_us_scalar=so, step_us_guided=sp, ratio=sp / so, rounds_scalar=one,
                              rounds_guided=per, card=card_s)), flush=True)

    out_u, out_c = banks[1].chunk(2)
    x_in = torch.empty((2 * B,) + SHAPE[1:], device="cuda", dtype=bf)
    step_case("c3_diff2_bf16_noise", ops.StepArgs(
        form=FORM_DIFF2, n_model=2, x=x, xe=x, m1=x, e_cond=out_c, e_uncond=out_u, guidance=7.5, a=0.9, c0=-0.1,
        c1=0.2, w0=1.0, c0_on_old=True, state_dtype=bf, out=x_in[:B], out2=x_in[B:]))
    del x_in
    f = torch.float32
    x32, m1, m2, ec, eu = (rnd(SHAPE, f) for _ in range(5))
    step_case("diff2_f32_v_x0", ops.StepArgs(
        form=FORM_DIFF2, n_model=2, x=x32, xe=x32, m1=m1, e_cond=ec, e_uncond=eu, guidance=7.5, param=PARAM_V,
        predict_x0=True, alpha_e=0.8, sigma_e=0.6, a=0.9, c0=-0.1, c1=0.2, w0=1.0, state_dtype=f))
    step_case("ss3t_f32_noise", ops.StepArgs(
        form=FORM_SS3T, n_model=2, x=x32, xe=x32, m1=m1, m2=m2, e_cond=ec, e_uncond=eu, guidance=7.5, a=0.9,
        c0=-0.1, c1=0.2, c2=0.1, w0=1.5, w1=0.7, w2=0.4, w3=0.6, w4=0.3, state_dtype=f))
    del x32, m1, m2, ec, eu
    torch.cuda.empty_cache()

    ns = NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    cnt = [0]

    def net(xx, tt, cc):
        cnt[0] += 1
        return banks[cnt[0] % 2]

    def sample_case(name, model_type, skw, **dkw):
        def solver(s):
            fn = model_wrapper(net, ns, model_type=model_type, guidance_type="classifier-free",
                               condition=torch.ones(B, 1, device="cuda"),
                               unconditional_condition=torch.zeros(B, 1, device="cuda"), guidance_scale=s)
            return DPM_Solver(fn, ns, state_dtype=bf, **dkw)
        runs = {"one": solver(7.5), "mixed": solver(scales)}
        dev = {k: [] for k in runs}
        host = {k: [] for k in runs}
        for s in runs.values():
            s.sample(x, **skw)
        for _ in range(args.samples):
            for k, s in runs.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record()
                s.sample(x, **skw)
                e1.record()
                host[k].append((time.perf_counter() - t0) * 1e6)
                torch.cuda.synchronize()
                dev[k].append(e0.elapsed_time(e1) * 1e3)
        med = lambda v: statistics.median(v)
        print(json.dumps(dict(case=name, sample_dev_us_one=med(dev["one"]), sample_dev_us_mixed=med(dev["mixed"]),
                              sample_host_us_one=med(host["one"]), sample_host_us_mixed=med(host["mixed"]),
                              dev_all=dev, host_all=host, card=card_s)), flush=True)

    sample_case("c3_sample", "noise", dict(steps=15, order=3, method="singlestep"), algorithm_type="dpmsolver")
    sample_case("v_thresholded_sample", "v", dict(steps=15, order=2, method="multistep"), algorithm_type="dpmsolver++",
                correcting_x0_fn="dynamic_thresholding")


if __name__ == "__main__":
    main()
