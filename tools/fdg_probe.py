"""Cost of frequency-decoupled guidance: the pyramid pass, the whole FDG evaluation and an eager-torch composition,
beside the plain CFG step, on bf16 network outputs and state.

    python tools/fdg_probe.py [--launches 60] [--rounds 5]

Shapes [2048,4,64,64], [4096,4,64,64] and [256,16,128,128]; levels N = 2 and 4; scales [10, 5] and [10, 5, 2.5, 1].
For each (shape, N) these are timed with CUDA events over `launches` launches that rotate over 3 buffer sets,
alternating within a round, the median of `rounds` rounds reported:
  - pass:   dpm_fdg_guided (1 launch), algorithmic bytes 3*s per element (c and u read, g written);
  - fdg:    the pass, then the one-output DIFF2 step on g (reads x, m1, g; writes x_t and the doubled next input),
            algorithmic bytes 3*s + 6*s;
  - cfg:    the plain CFG DIFF2 step on both halves (reads x, m1, c, u; writes x_t twice), 7*s;
  - eager:  the eager-torch per-level form (reflect pad, 5x5 binomial conv2d and bilinear resampling of both halves per
            level, the per-level combine and the reconstruction), then the same one-output step.
One JSON line per (shape, N) with us per call, GB/s over the algorithmic bytes and the ratio fdg/cfg, and the card's
name, power limit and maximum SM clock read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(2048, 4, 64, 64), (4096, 4, 64, 64), (256, 16, 128, 128)]
SCALES = {2: [10.0, 5.0], 4: [10.0, 5.0, 2.5, 1.0]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


_K = None


def _blur(x):
    global _K
    if _K is None or _K.device != x.device or _K.dtype != x.dtype:
        k1 = torch.tensor([1., 4., 6., 4., 1.], device=x.device) / 16
        _K = (k1[:, None] * k1[None, :]).to(x.dtype)[None, None]
    B, C, H, W = x.shape
    y = F.conv2d(F.pad(x.reshape(B * C, 1, H, W), (2, 2, 2, 2), mode="reflect"), _K)
    return y.reshape(B, C, H, W)


def eager_fdg(c, u, scales):
    """diffusers' per-level form in eager torch: Laplacian pyramids of both halves, combine per level, reconstruct."""
    def lap(x):
        G = [x]
        for _ in range(len(scales) - 1):
            G.append(F.interpolate(_blur(G[-1]), scale_factor=0.5, mode="bilinear", align_corners=False))
        up = lambda t: _blur(F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False))
        return [G[l] - up(G[l + 1]) for l in range(len(G) - 1)] + [G[-1]], up
    Lc, up = lap(c)
    Lu, _ = lap(u)
    L = [lu + w * (lc - lu) for lc, lu, w in zip(Lc, Lu, scales)]
    g = L[-1]
    for l in range(len(L) - 2, -1, -1):
        g = up(g) + L[l]
    return g


def run(shape, levels, launches, rounds):
    from dpm_solver_b200 import ops
    from dpm_solver_b200._lib import FORM_DIFF2
    be = ops.backend()
    B = shape[0]
    scales = SCALES[levels]
    g = torch.Generator(device="cuda").manual_seed(0)
    sets = []
    for _ in range(3):
        x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
        m1 = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16)
        bank = torch.randn((2 * B,) + shape[1:], device="cuda", generator=g).to(torch.bfloat16)
        out_u, out_c = bank.chunk(2)
        x_in = torch.empty((2 * B,) + shape[1:], device="cuda", dtype=torch.bfloat16)
        a = ops.StepArgs(form=FORM_DIFF2, n_model=2, x=x, xe=x, m1=m1, e_cond=out_c, e_uncond=out_u, param=0,
                         predict_x0=False, guidance=7.5, a=0.9, c0=-0.1, c1=0.2, w0=1.0, c0_on_old=True,
                         state_dtype=torch.bfloat16, out=x_in[:B], out2=x_in[B:])
        sets.append((a, out_c, out_u))

    def one_output(k, gout):
        a = ops.StepArgs(**{f: getattr(sets[k][0], f) for f in sets[k][0].__dataclass_fields__})
        a.n_model, a.e_cond, a.e_uncond, a.guidance = 1, gout, None, 1.0
        return be.step(a)

    n, s = sets[0][0].x.numel(), 2
    kernels = {
        "pass": (lambda k: be.fdg_guided(sets[k][1], sets[k][2], scales, levels), 3 * s * n),
        "fdg": (lambda k: one_output(k, be.fdg_guided(sets[k][1], sets[k][2], scales, levels)), 9 * s * n),
        "cfg": (lambda k: be.step(sets[k][0]), 7 * s * n),
        "eager": (lambda k: one_output(k, eager_fdg(sets[k][1], sets[k][2], scales)), 9 * s * n),
    }
    for fn, _ in kernels.values():          # warm every kernel and buffer set
        for k in range(3):
            fn(k)
    torch.cuda.synchronize()
    times = {k: [] for k in kernels}
    for _ in range(rounds):
        for key, (fn, _) in kernels.items():
            reps = launches if key != "eager" else max(1, launches // 6)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(reps):
                fn(i % 3)
            b.record()
            torch.cuda.synchronize()
            times[key].append(a.elapsed_time(b) * 1e3 / reps)
    res = dict(shape=list(shape), levels=levels, card=card())
    for key, (_, nbytes) in kernels.items():
        us = statistics.median(times[key])
        res[key + "_us"] = round(us, 1)
        res[key + "_gbs"] = round(nbytes / (us * 1e-6) / 1e9, 1)
        res[key + "_us_rounds"] = [round(t, 1) for t in times[key]]
    res["fdg_over_cfg"] = round(res["fdg_us"] / res["cfg_us"], 3)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fdg_probe measures on the GPU; no CUDA device found")
    with torch.no_grad():
        for shape in SHAPES:
            for levels in (2, 4):
                run(shape, levels, args.launches, args.rounds)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
