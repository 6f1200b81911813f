#!/usr/bin/env python
"""bench_multicond.py -- HBM throughput of the fused multi-condition CFG step on one GPU.

    python bench_multicond.py [--launches 60] [--rounds 5] [--sets 3] [--conds 2 4]

Times one DPM-Solver++ 2M multistep step (DIFF2, predict_x0) at bf16 [2048,4,64,64] with K conditions, on the same
synthetic network outputs three ways:
  fused : dpm_step_multi -- reads x, the K+1 network outputs and m1, writes m_out, x_t and the K replica blocks of the
          next [(K+1)B] network input: (2K+5)*s algorithmic bytes per element;
  eager : what a user writes today with guidance_type="uncond": the combine in the network's dtype with eager ATen ops
          (eu + s1*(e1 - eu) + ...), torch.cat([x] * (K+1)) for the next network input, then the fused one-output step;
  k1    : for comparison, the one-condition CFG step (dpm_step with out2), (2*1+5)*s bytes per element.
Each round times `launches` steps with two CUDA events, rotating over `sets` buffer sets (each far larger than L2) so that
no step reads what the previous one left in L2; after a warm-up of every set, rounds of the variants alternate and the
median round is reported. GB/s = algorithmic bytes / time; share = GB/s / 3350 GB/s (the H100 SXM data-sheet HBM3
bandwidth). The card's name, power limit and SM clock are read in the same run. Prints one JSON line per case.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SHAPE = (2048, 4, 64, 64)
PEAK_GBS = 3350.0
SCALES = [7.5, -2.0, 3.0, 0.5]
COEF = dict(a=0.9, c0=-0.1, c1=0.2, w0=1.3, alpha_e=0.8, sigma_e=0.6)


def card():
    pr = torch.cuda.get_device_properties(torch.cuda.current_device())
    bus = "%08X:%02X:%02X.0" % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
    q = subprocess.run(["nvidia-smi", "--id=" + bus, "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def time_round(fns, launches):
    """ms per launch of `launches` calls cycling over fns (one per buffer set), CUDA events around the whole loop."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(launches):
        fns[i % len(fns)]()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--conds", type=int, nargs="+", default=[2, 4])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multicond measures on the GPU; no CUDA device found")
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2
    torch.set_grad_enabled(False)
    be = ops.CudaBackend()
    bf = torch.bfloat16
    B, n = SHAPE[0], torch.Size(SHAPE).numel()
    s = 2
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda shape: torch.randn(shape, device="cuda", generator=g).to(bf)
    card_s = card()

    def report(case, K, ms_rounds, bytes_per_elem):
        ms = statistics.median(ms_rounds)
        gbs = bytes_per_elem * n / (ms * 1e-3) / 1e9
        print(json.dumps(dict(case=case, K=K, shape=list(SHAPE), dtype="bf16", us_per_step=ms * 1e3,
                              algorithmic_bytes_per_elem=bytes_per_elem, GBps=gbs, share_of_3350=gbs / PEAK_GBS,
                              rounds_us=[r * 1e3 for r in ms_rounds], launches_per_round=args.launches, card=card_s)),
              flush=True)

    for K in [1] + list(args.conds):
        sets = []
        for _ in range(args.sets):
            x, m1 = rnd(SHAPE), rnd(SHAPE)
            bank = rnd(((K + 1) * B,) + SHAPE[1:])
            x_in = torch.empty(((K + 1) * B,) + SHAPE[1:], device="cuda", dtype=bf)
            m_out = torch.empty(SHAPE, device="cuda", dtype=bf)
            sets.append((x, m1, bank, x_in, m_out))
        fused, eager = [], []
        for x, m1, bank, x_in, m_out in sets:
            outs = bank.chunk(K + 1)
            blocks = x_in.chunk(K + 1)
            base = dict(form=FORM_DIFF2, x=x, xe=x, m1=m1, predict_x0=True, state_dtype=bf, want_m_out=True,
                        m_out=m_out, out=blocks[0], **COEF)
            if K == 1:
                a = ops.StepArgs(n_model=2, e_cond=outs[1], e_uncond=outs[0], guidance=SCALES[0], out2=blocks[1], **base)
                fused.append(lambda a=a: be.step(a))
                continue
            a = ops.StepArgs(n_model=2, e_cond=outs[1], e_uncond=outs[0], e_conds=tuple(outs[1:]),
                             scales=tuple(SCALES[:K]), replicas=tuple(blocks[1:]), **base)
            fused.append(lambda a=a: be.step(a))

            def eager_step(x=x, outs=outs, base=base):
                e = outs[0]
                for sk, ek in zip(SCALES[:K], outs[1:]):
                    e = e + sk * (ek - outs[0])
                _, xt = be.step(ops.StepArgs(n_model=1, e_cond=e, **dict(base, out=None)))
                return torch.cat([xt] * (K + 1))
            eager.append(eager_step)
        variants = {"fused": fused} if K == 1 else {"fused": fused, "eager": eager}
        for fns in variants.values():
            for f in fns:
                f()
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fns in variants.items():
                times[k].append(time_round(fns, args.launches))
        if K == 1:
            report("k1_cfg_step", 1, times["fused"], (2 * 1 + 5) * s)
        else:
            report("fused_multi_step", K, times["fused"], (2 * K + 5) * s)
            report("eager_composition", K, times["eager"], (2 * K + 5) * s)
        del sets, fused, eager, variants
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
