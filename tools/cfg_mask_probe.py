"""Cost of the regional-guidance step (dpm_step_multi_masked) beside the unmasked multi-condition / CFG step.

    python tools/cfg_mask_probe.py [--launches 60] [--rounds 5]

Cases: one DPM-Solver++ 2M (DIFF2, predict_x0) step at bf16 state and outputs, [2048|4096,4,64,64], K = 1, 2 and 4
conditions, writing m, x_t and the K replica blocks of the next network input. Variants, alternating within a round:
  - shared:     every condition with a pixel map [H, W] shared by the batch (period H*W);
  - per_sample: every condition with a per-sample pixel map [B, 1, H, W];
  - unmasked:   dpm_step_multi for K >= 2, the plain CFG step (dpm_step with out2) for K = 1.
Algorithmic bytes (s = 2): (2K + 5)*s per element for every variant, plus 4K/C per element for the per-sample maps (a
shared map is read once per launch and then served by L2). Each variant is timed with CUDA events over `launches`
launches rotating over 3 buffer sets; the median of `rounds` rounds is reported. One JSON line per case with us per
launch and GB/s, and the card's name, power limit and SM clock read in the same run.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def run(shape, K, launches, rounds):
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2
    be = ops.backend()
    B, C, H, W = shape
    S = H * W
    g = torch.Generator(device="cuda").manual_seed(0)
    bf = torch.bfloat16
    sets = []
    for _ in range(3):
        x = torch.randn(shape, device="cuda", generator=g).to(bf)
        m1 = torch.randn(shape, device="cuda", generator=g).to(bf)
        outs = torch.randn(((K + 1) * B,) + shape[1:], device="cuda", generator=g).to(bf).chunk(K + 1)
        x_in = torch.empty(((K + 1) * B,) + shape[1:], device="cuda", dtype=bf)
        blocks = x_in.chunk(K + 1)
        m_out = torch.empty(shape, device="cuda", dtype=bf)
        base = dict(form=FORM_DIFF2, n_model=2, x=x, xe=x, m1=m1, e_cond=outs[1], e_uncond=outs[0], param=0,
                    predict_x0=True, a=0.9, c0=0.1, c1=-0.05, w0=1.2, alpha_e=0.8, sigma_e=0.6, state_dtype=bf,
                    out=blocks[0], m_out=m_out, want_m_out=True, per_sample=C * S)
        scales = tuple(7.5 / K for _ in range(K))
        shared = tuple((torch.rand(1, S, device="cuda", generator=g), S, 0) for _ in range(K))
        per_sample = tuple((torch.rand(B, S, device="cuda", generator=g), S, S) for _ in range(K))
        multi = dict(e_conds=tuple(outs[1:]), scales=scales, replicas=tuple(blocks[1:]))
        v = {"shared": ops.StepArgs(**base, **multi, masks=shared),
             "per_sample": ops.StepArgs(**base, **multi, masks=per_sample)}
        if K >= 2:
            v["unmasked"] = ops.StepArgs(**base, **multi)
        else:
            v["unmasked"] = ops.StepArgs(**base, guidance=scales[0], out2=blocks[1])
        sets.append(v)
    n, s = B * C * S, 2
    nbytes = {"shared": (2 * K + 5) * s * n, "unmasked": (2 * K + 5) * s * n,
              "per_sample": (2 * K + 5) * s * n + 4 * K * n // C}
    keys = list(sets[0])
    for key in keys:                     # warm every kernel and buffer set
        for k in range(3):
            be.step(sets[k][key])
    torch.cuda.synchronize()
    times = {k: [] for k in keys}
    for _ in range(rounds):
        for key in keys:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(launches):
                be.step(sets[i % 3][key])
            b.record()
            torch.cuda.synchronize()
            times[key].append(a.elapsed_time(b) * 1e3 / launches)
    res = dict(shape=list(shape), K=K, card=card())
    for key in keys:
        us = statistics.median(times[key])
        res[key + "_us"] = round(us, 1)
        res[key + "_gbs"] = round(nbytes[key] / (us * 1e-6) / 1e9, 1)
        res[key + "_us_rounds"] = [round(t, 1) for t in times[key]]
    res["shared_over_unmasked_time"] = round(res["shared_us"] / res["unmasked_us"], 4)
    res["per_sample_over_unmasked_gbs"] = round(res["per_sample_gbs"] / res["unmasked_gbs"], 4)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cfg_mask_probe measures on the GPU; no CUDA device found")
    with torch.no_grad():
        for shape in ((2048, 4, 64, 64), (4096, 4, 64, 64)):
            for K in (1, 2, 4):
                run(shape, K, args.launches, args.rounds)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
