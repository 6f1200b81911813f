"""Cost of the CFG++ step beside the plain CFG step it replaces, on the benchmark's CFG shapes.

    python tools/cfgpp_probe.py [--launches 60] [--rounds 5]

Cases (bf16 state and network outputs, the DPM-Solver++ 2M update of a multistep run):
  - noise_2048 / noise_4096: [2048|4096,4,64,64], eps network;
  - flow_2048 / flow_4096:   the same shapes, flow network.
Both kernels read x, m1 and both halves and write m, x_t and the doubled next input: 7*s algorithmic bytes per element.
  - cfgpp: dpm_step_cfgpp (m receives U, the x0 of the unconditional half alone);
  - cfg:   the plain CFG DIFF2 step (dpm_step, m receives the guided x0).
Each is timed with CUDA events over `launches` launches that rotate over 3 buffer sets, the two kernels alternating within
a round, the median of `rounds` rounds reported. One JSON line per case with us per launch and GB/s of the 7*s bytes, and
the card's name and power limit read in the same run.
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

CASES = {
    "noise_2048": dict(shape=(2048, 4, 64, 64), param=0),
    "noise_4096": dict(shape=(4096, 4, 64, 64), param=0),
    "flow_2048": dict(shape=(2048, 4, 64, 64), param=4),
    "flow_4096": dict(shape=(4096, 4, 64, 64), param=4),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def run(name, c, launches, rounds):
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2
    be = ops.backend()
    shape, B = c["shape"], c["shape"][0]
    g = torch.Generator(device="cuda").manual_seed(0)
    sets = []
    for _ in range(3):
        x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
        m1 = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
        bank = torch.randn((2 * B,) + shape[1:], device="cuda", generator=g).to(torch.bfloat16)
        out_u, out_c = bank.chunk(2)
        x_in = torch.empty((2 * B,) + shape[1:], device="cuda", dtype=torch.bfloat16)
        m_out = torch.empty(shape, device="cuda", dtype=torch.bfloat16)
        a = ops.StepArgs(form=FORM_DIFF2, n_model=2, x=x, xe=x, m1=m1, e_cond=out_c, e_uncond=out_u,
                         param=c["param"], predict_x0=True, guidance=0.6, a=0.9, c0=0.1, c1=-0.05, w0=1.2,
                         state_dtype=torch.bfloat16, alpha_e=0.8, sigma_e=0.6, out=x_in[:B], out2=x_in[B:],
                         m_out=m_out, want_m_out=True)
        p = ops.StepArgs(**{k: getattr(a, k) for k in a.__dataclass_fields__})
        p.cfgpp_g = 0.8
        sets.append((a, p))
    n, s = sets[0][0].x.numel(), 2
    step_bytes = s * n * 7          # x, m1, two halves read; m, x_t twice written
    kernels = {
        "cfgpp": lambda k: be.step(sets[k][1]),
        "cfg": lambda k: be.step(sets[k][0]),
    }
    for fn in kernels.values():          # warm every kernel and buffer set
        for k in range(3):
            fn(k)
    torch.cuda.synchronize()
    times = {k: [] for k in kernels}
    for _ in range(rounds):
        for key, fn in kernels.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(launches):
                fn(i % 3)
            b.record()
            torch.cuda.synchronize()
            times[key].append(a.elapsed_time(b) * 1e3 / launches)
    res = dict(case=name, shape=list(shape), card=card())
    for key in kernels:
        us = statistics.median(times[key])
        res[key + "_us"] = round(us, 1)
        res[key + "_gbs"] = round(step_bytes / (us * 1e-6) / 1e9, 1)
        res[key + "_us_rounds"] = [round(t, 1) for t in times[key]]
    res["cfgpp_over_cfg"] = round(res["cfgpp_us"] / res["cfg_us"], 4)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cfgpp_probe measures on the GPU; no CUDA device found")
    with torch.no_grad():
        for name, c in CASES.items():
            run(name, c, args.launches, args.rounds)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
