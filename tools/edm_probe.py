"""Cost of the EDM parameterisation on the benchmark's step shapes.

    python tools/edm_probe.py [--launches 60] [--sets 3] [--rounds 5]

At c2's step (bf16 [4096,4,64,64], DPM-Solver++ 2M: one DIFF2 launch that reads x, the network output and the older
buffer and writes the model value and x_t) and at c3's (bf16 [2048,4,64,64], eps-solver, CFG 7.5: the same launch with
two network outputs), times the step of an EDM network (DPM_PARAM_EDM, with the words of each space), of a noise network
(DPM_PARAM_NOISE) and of a flow network (DPM_PARAM_FLOW, which shares EDM's conversion code) in one process, alternating
between them: CUDA events over `launches` launches that rotate through `sets` buffer sets (so no
launch finds its operands in L2), the median of `rounds` rounds. Prints one JSON line per case with the two times in
microseconds, the rate in GB/s over the algorithmic bytes (equal for all: 5 or 6 tensors of the shape), and the card's
name, power limit and SM clock read in the same run.
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
    "c2_step": dict(shape=(4096, 4, 64, 64), predict_x0=True, cfg=False),
    "c3_step": dict(shape=(2048, 4, 64, 64), predict_x0=False, cfg=True),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def run(name, c, launches, sets, rounds):
    from dpm_solver_b200 import ops
    from dpm_solver_b200 import NoiseScheduleEDM
    from dpm_solver_b200._lib import FORM_DIFF2, PARAM_EDM, PARAM_FLOW, PARAM_NOISE
    from dpm_solver_b200.ops import StepArgs
    be = ops.backend()
    shape, bf16 = c["shape"], torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(0)
    new = lambda: torch.randn(shape, device="cuda", generator=g).to(bf16)
    # EDM's words at sigma = 2.5 (alpha_t = 0.392, sigma_t = 0.981) in the launch's space
    ew = NoiseScheduleEDM().conversion_words(0.392, 0.981, c["predict_x0"])
    words = {"edm": ew, "noise": (0.4, 0.6), "flow": (0.4, 0.6)}
    steps = {"edm": [], "noise": [], "flow": []}
    for _ in range(sets):
        x, m1, ec, eu = new(), new(), new(), new() if c["cfg"] else None
        m_out, out = torch.empty_like(x), torch.empty_like(x)
        for label, param in (("edm", PARAM_EDM), ("noise", PARAM_NOISE), ("flow", PARAM_FLOW)):
            steps[label].append(StepArgs(form=FORM_DIFF2, n_model=2 if c["cfg"] else 1, x=x, m1=m1, e_cond=ec, e_uncond=eu,
                                         guidance=7.5, param=param, predict_x0=c["predict_x0"], alpha_e=words[label][0],
                                         sigma_e=words[label][1],
                                         a=0.9, c0=-0.3, c1=0.2, w0=1.5, want_m_out=True, state_dtype=bf16, m_out=m_out,
                                         out=out))

    def timed(label):
        args = steps[label]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(launches):
            be.step(args[i % sets])
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) * 1e3 / launches

    for label in steps:                 # warm-up: module load, every buffer set touched
        timed(label)
    us = {label: [] for label in steps}
    for _ in range(rounds):
        for label in steps:
            us[label].append(timed(label))
    n = 1
    for d in shape:
        n *= d
    nbytes = n * 2 * (6 if c["cfg"] else 5)
    res = dict(case=name, shape=list(shape), launches=launches, buffer_sets=sets, rounds=rounds, bytes=nbytes, card=card())
    for label, v in us.items():
        med = statistics.median(v)
        res[label + "_us"] = round(med, 1)
        res[label + "_gbs"] = round(nbytes / med / 1e3, 1)
        res[label + "_us_min_max"] = [round(min(v), 1), round(max(v), 1)]
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("edm_probe needs a CUDA device")
    for name, c in CASES.items():
        run(name, c, a.launches, a.sets, a.rounds)


if __name__ == "__main__":
    main()
