"""Cost of the fused UniPC step on the benchmark's step shapes, and of UniPC sampling.

    python tools/unipc_probe.py [--launches 60] [--sets 3] [--rounds 5]

* c2_step: bf16 [4096,4,64,64], noise network, dpmsolver++. The fused UniPC-2 launch (corrector of order 2 and
  predictor of order 2: reads x~, eps, m_{i-1}, m_{i-2}, writes m_i and x~_{i+1}, 6 tensors) against the DPM-Solver++ 2M
  DIFF2 launch (reads x, eps, m1, writes m and x_t, 5 tensors), alternating between them in one process.
* c3_step: bf16 [2048,4,64,64], eps-solver, CFG 7.5: the same two launches with two network outputs and the doubled
  batch written (8 and 7 tensors).
* eager_step: the same UniPC-2 step at c2 as separate torch ops (conversion, corrector, predictor), the baseline.
* sample_20: UniPC(order 2) against DPM_Solver(multistep, order 2), 20 steps at [8,4,64,64] bf16 state, a trivial
  network, device time of a whole sample() call.
Every time is the median of `rounds` rounds of CUDA events over `launches` launches that rotate through `sets` buffer
sets (so no launch finds its operands in L2), with the min and max; the rate is over the algorithmic bytes. The card's
name, power limit and SM clock are read in the same run.
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, launches):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(launches):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / launches


def compare(name, fns, launches, rounds, nbytes, extra=None):
    for f in fns.values():
        timed(f, launches)                                  # warm-up: module load, every buffer set touched
    us = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            us[k].append(timed(f, launches))
    res = dict(case=name, launches=launches, rounds=rounds, card=card())
    res.update(extra or {})
    for k, v in us.items():
        med = statistics.median(v)
        res[k + "_us"] = round(med, 1)
        res[k + "_us_min_max"] = [round(min(v), 1), round(max(v), 1)]
        if nbytes.get(k):
            res[k + "_gbs"] = round(nbytes[k] / med / 1e3, 1)
    print(json.dumps(res), flush=True)


def steps(shape, cfg, sets):
    from dpm_solver_b200 import plan as P
    from dpm_solver_b200._lib import FORM_DIFF2, PARAM_NOISE
    from dpm_solver_b200.ops import StepArgs
    bf16 = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(0)
    new = lambda: torch.randn(shape, device="cuda", generator=g).to(bf16)
    w = P.UniCoeffs(2, 2, (0.4375, 0.0), -0.8125, 0.96875, -0.15625, (0.3125, 0.0))
    uni, diff2, eager = [], [], []
    for _ in range(sets):
        x, m1, m2, ec = new(), new(), new(), new()
        eu = new() if cfg else None
        m_out, out, out2 = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x) if cfg else None
        common = dict(n_model=2 if cfg else 1, x=x, e_cond=ec, e_uncond=eu, guidance=7.5, param=PARAM_NOISE,
                      predict_x0=not cfg, alpha_e=0.4, sigma_e=0.6, want_m_out=True, state_dtype=bf16, m_out=m_out,
                      out=out, out2=out2)
        uni.append(StepArgs(form=1, m1=m1, m2=m2, unipc=w, **common))
        diff2.append(StepArgs(form=FORM_DIFF2, m1=m1, a=0.9, c0=-0.3, c1=0.2, w0=1.5, **common))
        eager.append((x, ec, m1, m2))
    return w, uni, diff2, eager


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("unipc_probe needs a CUDA device")
    from dpm_solver_b200 import DPM_Solver, NoiseScheduleVP, UniPC, model_wrapper, ops
    from cases import make_betas
    be = ops.backend()
    for name, shape, cfg in (("c2_step", (4096, 4, 64, 64), False), ("c3_step", (2048, 4, 64, 64), True)):
        w, uni, diff2, eager = steps(shape, cfg, a.sets)
        n = 1
        for d in shape:
            n *= d
        fns = {"unipc2": lambda i: be.step(uni[i % a.sets]), "dpmpp_2m": lambda i: be.step(diff2[i % a.sets])}
        nbytes = {"unipc2": n * 2 * (8 if cfg else 6), "dpmpp_2m": n * 2 * (7 if cfg else 5)}
        if not cfg:
            def eager_step(i, e=eager):
                x, ec, m1, m2 = e[i % a.sets]
                T = ((x.float() - 0.6 * ec.float()) / 0.4).to(torch.bfloat16).float()
                c = x.float() + w.cd[0] * (m2.float() - m1.float())
                c = (c + w.ct * (T - m1.float())).to(torch.bfloat16).float()
                o = w.a * c + w.c0 * T
                return (o + w.cp[0] * (m1.float() - T)).to(torch.bfloat16)
            fns["eager_unipc2"] = eager_step
            nbytes["eager_unipc2"] = n * 2 * 6
        compare(name, fns, a.launches, a.rounds, nbytes, dict(shape=list(shape), buffer_sets=a.sets))
        del uni, diff2, eager
        torch.cuda.empty_cache()

    ns = NoiseScheduleVP("discrete", betas=torch.from_numpy(make_betas("sd")[1]))
    net = lambda x, t: 0.1 * x
    x = torch.randn(8, 4, 64, 64, device="cuda")
    u = UniPC(model_wrapper(net, ns), ns, state_dtype=torch.bfloat16)
    d = DPM_Solver(model_wrapper(net, ns), ns, state_dtype=torch.bfloat16)
    fns = {"unipc2_sample": lambda i: u.sample(x, steps=20, order=2),
           "dpmpp_2m_sample": lambda i: d.sample(x, steps=20, order=2, method="multistep")}
    compare("sample_20", fns, 10, a.rounds, {}, dict(shape=[8, 4, 64, 64]))


if __name__ == "__main__":
    main()
