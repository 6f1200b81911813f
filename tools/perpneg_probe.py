"""Cost of Perp-Neg on the benchmark's shape: the words pass for K = 2, 3, 4 beside the TCFG words pass, and the K = 2
Perp-Neg step beside the plain multi-condition step.

    python tools/perpneg_probe.py [--launches 60] [--rounds 5]

bf16 network outputs and state, [2048,4,64,64]. Kernels timed with CUDA events over `launches` launches that rotate over
3 buffer sets, all kernels alternating within a round, the median of `rounds` rounds reported:
  - pass_k{K}:  dpm_perpneg_words (2 launches), algorithmic bytes (K+1)*s per element;
  - tcfg_pass:  dpm_tcfg_words (2 launches) on two of the blocks, 2*s per element (the streaming rate to compare with);
  - perpneg:    dpm_step_multi_masked with scales (1, s_2) and the words as condition 1's period-1 map, K = 2;
  - multi:      dpm_step_multi with the same outputs and scales (s_1, s_2), K = 2.
Both steps are the DPM-Solver-3 singlestep difference step of an eps network: they read x, m1 and the 3 blocks and
write x_t into the 3 blocks of the next network input, 8*s bytes per element. One JSON line with us per launch and GB/s,
and the card's name, power limit and maximum SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPE = (2048, 4, 64, 64)
SCALES = {2: [7.5, -3.0], 3: [7.5, -3.0, -2.0], 4: [7.5, -3.0, -2.0, -1.0]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def run(launches, rounds):
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2
    be = ops.backend()
    B = SHAPE[0]
    g = torch.Generator(device="cuda").manual_seed(0)
    sets = []
    for _ in range(3):
        x = torch.randn(SHAPE, device="cuda", generator=g).to(torch.bfloat16)
        m1 = torch.randn(SHAPE, device="cuda", generator=g).to(torch.bfloat16)
        bank = torch.randn((5 * B,) + SHAPE[1:], device="cuda", generator=g).to(torch.bfloat16)
        blocks = bank.chunk(5)                          # u, e_1 .. e_4
        x_in = torch.empty((3 * B,) + SHAPE[1:], device="cuda", dtype=torch.bfloat16)
        words = be.perpneg_words(blocks[0], blocks[1:3], SCALES[2])
        base = dict(form=FORM_DIFF2, n_model=2, x=x, xe=x, m1=m1, e_cond=blocks[1], e_uncond=blocks[0], param=0,
                    a=0.9, c0=-0.1, c1=0.2, w0=1.0, c0_on_old=True, state_dtype=torch.bfloat16,
                    out=x_in[:B], e_conds=tuple(blocks[1:3]), replicas=(x_in[B:2 * B], x_in[2 * B:]))
        multi = ops.StepArgs(scales=tuple(SCALES[2]), **base)
        perp = ops.StepArgs(scales=(1.0, SCALES[2][1]), masks=((words, 1, 1), None), per_sample=x.numel() // B,
                            **base)
        sets.append((blocks, multi, perp))
    n, s = sets[0][1].x.numel(), 2
    kernels = {}
    for K in (2, 3, 4):
        kernels["pass_k%d" % K] = (lambda k, K=K: be.perpneg_words(sets[k][0][0], sets[k][0][1:K + 1], SCALES[K]),
                                   (K + 1) * s * n)
    kernels["tcfg_pass"] = (lambda k: be.tcfg_words(sets[k][0][1], sets[k][0][0]), 2 * s * n)
    kernels["perpneg"] = (lambda k: be.step(sets[k][2]), 8 * s * n)
    kernels["multi"] = (lambda k: be.step(sets[k][1]), 8 * s * n)
    for fn, _ in kernels.values():          # warm every kernel and buffer set
        for k in range(3):
            fn(k)
    torch.cuda.synchronize()
    times = {k: [] for k in kernels}
    for _ in range(rounds):
        for key, (fn, _) in kernels.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(launches):
                fn(i % 3)
            b.record()
            torch.cuda.synchronize()
            times[key].append(a.elapsed_time(b) * 1e3 / launches)
    res = dict(shape=list(SHAPE), card=card())
    for key, (_, nbytes) in kernels.items():
        us = statistics.median(times[key])
        res[key + "_us"] = round(us, 1)
        res[key + "_gbs"] = round(nbytes / (us * 1e-6) / 1e9, 1)
        res[key + "_us_rounds"] = [round(t, 1) for t in times[key]]
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perpneg_probe measures on the GPU; no CUDA device found")
    with torch.no_grad():
        run(args.launches, args.rounds)


if __name__ == "__main__":
    main()
