#!/usr/bin/env python
"""Replay the launch sequence of bench.py's c2 workload (DPM-Solver++ 2M, 20 steps, bf16 [4096,4,64,64]) with its
data flow, and time it per step and per chain for a list of launch shapes.

    python tools/c2_chain_probe.py                        # variant 0 (direct) and 1 (TMA) at their defaults
    python tools/c2_chain_probe.py --sweep                # + threads x CTAs/SM of both variants
    python tools/c2_chain_probe.py --configs 0:256:0,1:0:0

One chain = LIN1 (eps in, x_t and the model value stored), 18 x DIFF2 (model value stored), DIFF2 without the stored
value; x_{i+1} = out_i, m1 = m_out_i, eps from 3 rotating bf16 banks, outputs freshly allocated by the library's
backend as the solver does. Per-step times come from CUDA events around each launch over --chains chains; the chain
time from events around whole chains without per-launch events (those keep consecutive launches from overlapping).
Rates are algorithmic bytes (streams read + written) over time, against --peak GB/s (H100 SXM data sheet: 3350).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from dpm_solver_b200 import ops  # noqa: E402
from dpm_solver_b200._lib import FORM_DIFF2, FORM_LIN1  # noqa: E402
from dpm_solver_b200.ops import StepArgs  # noqa: E402

STEPS = 20


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:
        return f"unknown ({e!r:.80})"


def chain(be, x, banks, events):
    """One c2 sample(): returns the final x; with `events`, appends (kind, start, end) per launch."""
    m1 = None
    for i in range(STEPS):
        first, last = i == 0, i == STEPS - 1
        a = StepArgs(form=FORM_LIN1 if first else FORM_DIFF2, n_model=1, predict_x0=True, alpha_e=0.83 - 0.01 * i,
                     sigma_e=0.55 + 0.01 * i, a=0.95, c0=-0.1, c1=0.05, w0=1.02, want_m_out=not last,
                     x=x, xe=x, e_cond=banks[i % 3], m1=m1)
        if events is not None:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
        m_new, x = be.step(a)
        if events is not None:
            e.record()
            events.append(("lin1" if first else "diff2_last" if last else "diff2", s, e))
        m1 = m_new
    return x


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def measure(be, x0, banks, n, chains, peak):
    for _ in range(3):
        chain(be, x0, banks, None)
    torch.cuda.synchronize()
    ev = []
    for _ in range(chains):
        chain(be, x0, banks, ev)
    ce = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(chains)]
    for s, e in ce:
        s.record()
        chain(be, x0, banks, None)
        e.record()
    torch.cuda.synchronize()
    row = {}
    for kind, bpe in (("lin1", 8), ("diff2", 10), ("diff2_last", 8)):
        us = median([s.elapsed_time(e) * 1e3 for k, s, e in ev if k == kind])
        gbs = bpe * n / us / 1e3
        row[kind] = dict(us=round(us, 1), gbs=round(gbs), frac=round(gbs / peak, 3))
    us = median([s.elapsed_time(e) * 1e3 for s, e in ce])
    b = (8 + 18 * 10 + 8) * n
    row["chain"] = dict(us=round(us, 1), gbs=round(b / us / 1e3), frac=round(b / us / 1e3 / peak, 3))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="4096,4,64,64")
    ap.add_argument("--chains", type=int, default=20)
    ap.add_argument("--configs", default="0:0:0,1:0:0", help="variant:threads:ctas_per_sm, comma separated")
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--label", default="")
    ap.add_argument("--peak", type=float, default=3350.0)
    a = ap.parse_args()
    n = 1
    for v in a.shape.split(","):
        n *= int(v)
    cfgs = [tuple(int(v) for v in c.split(":")) for c in a.configs.split(",")]
    if a.sweep:
        cfgs += [(0, t, c) for t in (128, 256, 512) for c in (1, 2, 3, 4, 6, 8) if t * c <= 2048]
        cfgs += [(1, t, c) for t, c in ((256, 1), (256, 2), (128, 2), (128, 3), (512, 1))]
    print(json.dumps(dict(card=card(), label=a.label, shape=a.shape)), flush=True)
    be = ops.CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    banks = [torch.randn(n, device="cuda", generator=g).bfloat16() for _ in range(3)]
    x0 = torch.randn(n, device="cuda", generator=g).bfloat16()
    for variant, threads, ctas in cfgs:
        be.set_tuning(variant, threads, ctas)
        row = measure(be, x0, banks, n, a.chains, a.peak)
        print(json.dumps(dict(label=a.label, variant=variant, threads=threads, ctas=ctas, **row)), flush=True)
    be.set_tuning(2, 0, 0)


if __name__ == "__main__":
    main()
