"""Cost of TCFG on the benchmark's CFG shapes: the TCFG words pass and step beside the CFG-Zero* s* pass and step and
the plain CFG step.

    python tools/tcfg_probe.py [--launches 60] [--rounds 5]

Cases (bf16 state and network outputs):
  - c3:       [2048,4,64,64], eps network, CFG 7.5, the DPM-Solver-3 singlestep difference step (reads x, m1, both halves;
              writes x_t and the doubled next input);
  - flow_2m:  [4096,4,64,64], flow network, CFG 5.0, the DPM-Solver++ 2M step (reads x, m1, both halves; writes m,
              x_t and the doubled next input).
For each case five kernels are timed with CUDA events over `launches` launches that rotate over 3 buffer sets, the
five kernels alternating within a round, the median of `rounds` rounds reported:
  - tcfg_pass:    dpm_tcfg_words (2 launches), algorithmic bytes 2*s per element;
  - tcfg:         dpm_step_tcfg, bytes of the matching CFG step;
  - cfgzero_pass: dpm_cfgzero_scale (2 launches), 2*s per element;
  - cfgzero:      dpm_step_cfgzero, bytes of the matching CFG step;
  - cfg:          the plain CFG step (dpm_step), the same bytes.
One JSON line per case with us per launch and GB/s, and the card's name, power limit and maximum SM clock read in the
same run.
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
    "c3": dict(shape=(2048, 4, 64, 64), param=0, px0=False, guidance=7.5, want_m=False),
    "flow_2m": dict(shape=(4096, 4, 64, 64), param=4, px0=True, guidance=5.0, want_m=True),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
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
        m_out = torch.empty(shape, device="cuda", dtype=torch.bfloat16) if c["want_m"] else None
        a = ops.StepArgs(form=FORM_DIFF2, n_model=2, x=x, xe=x, m1=m1, e_cond=out_c, e_uncond=out_u,
                         param=c["param"], predict_x0=c["px0"], guidance=c["guidance"], a=0.9, c0=-0.1, c1=0.2,
                         w0=1.0, c0_on_old=True, state_dtype=torch.bfloat16, alpha_e=0.8, sigma_e=0.6,
                         out=x_in[:B], out2=x_in[B:], m_out=m_out, want_m_out=c["want_m"])
        z = ops.StepArgs(**{k: getattr(a, k) for k in a.__dataclass_fields__})
        z.per_sample = x.numel() // B
        z.cfgzero_s = be.cfgzero_scale(out_c, out_u)
        t = ops.StepArgs(**{k: getattr(a, k) for k in a.__dataclass_fields__})
        t.per_sample = z.per_sample
        t.tcfg_w = be.tcfg_words(out_c, out_u)
        sets.append((a, z, t))
    n, s = sets[0][0].x.numel(), 2
    step_bytes = s * n * (4 + 2 + (1 if c["want_m"] else 0))     # x, m1, two halves; x_t twice (+ m)
    kernels = {
        "tcfg_pass": (lambda k: be.tcfg_words(sets[k][0].e_cond, sets[k][0].e_uncond), 2 * s * n),
        "tcfg": (lambda k: be.step(sets[k][2]), step_bytes),
        "cfgzero_pass": (lambda k: be.cfgzero_scale(sets[k][0].e_cond, sets[k][0].e_uncond), 2 * s * n),
        "cfgzero": (lambda k: be.step(sets[k][1]), step_bytes),
        "cfg": (lambda k: be.step(sets[k][0]), step_bytes),
    }
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
    res = dict(case=name, shape=list(shape), card=card())
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
        raise SystemExit("tcfg_probe measures on the GPU; no CUDA device found")
    with torch.no_grad():
        for name, c in CASES.items():
            run(name, c, args.launches, args.rounds)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
