"""Random SDE-DPM-Solver++ `sample()` configurations for the end-to-end tests on the device
(tests/test_gpu_sde_random_configs.py) and their CPU side (tests/test_sde_draws_vs_reference.py): the draw
(apg_configs.draw_apg's base), an `SdeRig` and the oracle.

The base is draw_apg's: VP, flow and EDM schedules, every model type, 35 to 16384 elements per sample, B from 1 to 4, a
channels_last x_T, networks whose outputs keep their input's layout or are channels_last or row-major, 16-bit state
and model dtypes, thresholding, denoise_to_zero, t_start / t_end, skip types and lower_order_final. Then
algorithm_type="sde-dpmsolver++", multistep of order 1-3, either solver type, eta from {0, 0.5, 1, 2}, the generator
an explicit one on x's device or None (the device's default generator, seeded), and guidance: none, a scalar, a
one-element tensor or per-sample scales, the rescale, CFG-Zero*, TCFG or FDG. Now and then a configuration the SDE
solver refuses (REFUSALS): singlestep, adaptive, inverse(), UniPC, several conditions, a mask, Perp-Neg, APG, CFG++,
reference_rounding, a bad eta, or a generator that is not one on x's device (on the CPU, where no other device's
generator exists, an object that is not a generator).

The oracle of a configuration: the product's host logic on `SdeOracle` with the rig's tensors on the run's device, so
that each update's z is the contract's draw `torch.empty_like(x, dtype=float32).normal_(generator=g)` from the same
generator -- y, every intermediate, the trace of network calls and the generator's final offset, what the device must
give bit for bit. Two pins:
  * eta = 0: the run is the same configuration under algorithm_type="dpmsolver++" bit for bit and draws nothing;
  * where sde_oracle.kdiff_sde can express the draw (fp32, no guidance and no thresholding, no denoise_to_zero, a
    network with a closed-form x0 on a VP or flow schedule, order 3 with the "taylor" warm-up, and no lowered final
    order), the executor lies within KDIFF_TOL of the float64 k-diffusion loop fed `SdeOracle.draws`.
"""
import random

import numpy as np
import torch

from apg_configs import APGRig, draw_apg, per_sample
from gpu_configs import backend, really_channels_last, same_bits
from guidance_configs import VP, GuidanceRig, draw_fdg
from sde_oracle import SdeOracle, kdiff_sde

ETAS = [0.0, 0.5, 1.0, 2.0]
GUIDANCE = ["none", "none", "none", "float", "tensor0", "per_sample", "rescale", "cfgzero", "tcfg", "tcfg", "fdg"]
REFUSALS = ("singlestep", "adaptive", "inverse", "unipc", "multi", "mask", "perp", "apg", "cfgpp", "rr", "eta",
            "generator")
KDIFF_TOL = 2e-5              # tests/test_sde.py's bound against the float64 loop
CHUNKS, PER_CHUNK, SEED = 8, 20, 10400    # the device test: 8 chunks of 20 configurations


def draw_sde(rng):
    c = draw_apg(rng)
    c.update(apg_eta=None, apg_thr="off", apg_momentum=0.0, phi=0.0, tuning="auto", sampler="dpm", method="multistep",
             algo="sde-dpmsolver++", inverse=False, reference_rounding=False, zero_init=0, K=0, masks=None,
             perp_refusal=None, perp_d1_zero=None, cfgpp_refusal=None, fdg_levels=0, fdg_form=None, fdg_w=None,
             fdg_equal=False)
    if c["schedule"] in ("flow", "edm") and rng.random() < 0.4:
        c.update(schedule=rng.choice(VP), model_type=rng.choice(["noise", "x_start", "v", "score"]))
    c["order"] = rng.choice([1, 2, 3])
    c["solver_type"] = rng.choice(["dpmsolver", "taylor"])
    c["steps"] = max(min(c["steps"], 12), c["order"])
    c["eta"] = rng.choice(ETAS)
    c["generator"] = rng.choice(["explicit", "default"])
    B = c["B"]
    g = c["guidance"] = rng.choice(GUIDANCE)
    c["feature"] = g if g in ("cfgzero", "tcfg", "fdg") else "plain"
    c["cfg"], c["scales"] = None, None
    if g in ("float", "rescale", "cfgzero", "tcfg", "tensor0"):
        c["cfg"] = rng.choice([1.0, 3.5, 7.5, 7.5])
    if g == "per_sample" or (g in ("cfgzero", "tcfg") and rng.random() < 0.3):
        rows = [rng.choice([7.5, 1.0, 3.5, -2.0]) for _ in range(B)]
        c.update(guidance="per_sample", cfg=None, scales=rows)
    if g == "rescale":
        c.update(guidance="float", phi=0.7)
    if g == "cfgzero":
        c["zero_init"] = rng.choice([0, 1, 2])
    if g == "tcfg" and rng.random() < 0.3:
        c["thresholding"] = True             # (TCFG with thresholding materialises g before the step)
    if g == "fdg":
        draw_fdg(rng, c)
    c["refusal"] = None
    if rng.random() < 0.2:
        why = c["refusal"] = rng.choice(REFUSALS)
        c.update({"singlestep": dict(method=rng.choice(["singlestep", "singlestep_fixed"])),
                  "adaptive": dict(method="adaptive", atol=0.0078, rtol=0.05),
                  "inverse": dict(inverse=True, t_start=None, t_end=None),
                  "unipc": dict(sampler="unipc", variant="bh2", use_corrector=False),
                  "multi": dict(feature="plain", guidance="multi", cfg=None, scales=[3.5, -1.0]),
                  "mask": dict(feature="mask", guidance="multi", K=1, masks=[("b111", "f32")], cfg=None, scales=[3.5]),
                  "perp": dict(feature="perp", guidance="perp", K=2, cfg=None, scales=[7.5, -2.5]),
                  "apg": dict(feature="plain", guidance="float", cfg=3.5, apg_eta=0.3),
                  "cfgpp": dict(feature="cfgpp", guidance="float", cfg=0.6, scales=None),
                  "rr": dict(reference_rounding=True),
                  "eta": dict(eta=rng.choice([-1.0, float("nan"), float("inf"), True])),
                  "generator": dict(generator="foreign")}[why])
    return c


class SdeRig(GuidanceRig):
    """The configuration's schedule, network, model_fn and SDE solver (GuidanceRig for CFG-Zero*, TCFG, FDG and the
    refused multi-condition forms, APGRig else), sampled with its eta and a generator."""

    def __init__(self, mod, c, device="cpu"):
        if c["feature"] in ("cfgzero", "tcfg", "fdg", "mask", "perp", "cfgpp"):
            GuidanceRig.__init__(self, mod, c, device)
        else:
            APGRig.__init__(self, mod, c, device)

    def generator(self, seed):
        """The run's generator, seeded: explicit (a torch.Generator on x's device), or None with the device's default
        generator seeded; "foreign": one on another device (the CPU's on a CUDA device, else not a generator)."""
        kind, dev = self.c["generator"], self.device
        if kind == "explicit":
            return torch.Generator(dev).manual_seed(seed)
        if kind == "foreign":
            return torch.Generator().manual_seed(seed) if dev.type == "cuda" else seed
        default_generator(dev).manual_seed(seed)
        return None

    def sample(self, s, x, trace=False, gen=None, **over):
        c = self.c
        if c["sampler"] == "unipc" or c["inverse"] or c["method"] == "adaptive":
            return super().sample(s, x, trace, **over)
        return super().sample(s, x, trace, eta=c["eta"], generator=gen, **over)


def default_generator(dev):
    dev = torch.device(dev)
    if dev.type == "cuda":
        return torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
    return torch.default_generator


def refused(c):
    """Whether the product must refuse `c` with a ValueError before any launch."""
    if c["schedule"] == "flow" and c["model_type"] in ("v", "score"):
        return True
    if c["refusal"] is not None:
        return True
    if c["feature"] == "fdg":
        from guidance_configs import fdg_max_levels
        return c["fdg_levels"] > fdg_max_levels(c["shape"]) or c["fdg_form"] == "bad_rows"
    return False


# ---- the oracle ------------------------------------------------------------------------------------------------------

def kdiff_expressible(c):
    """fp32, no guidance, no thresholding, no denoise_to_zero, a closed-form x0 on a VP or flow schedule, order 3 only
    with the Heun warm-up, and the final order not lowered."""
    if refused(c) or c["state_dtype"] or c["model_dtype"] or c["guidance"] != "none" or c["thresholding"]:
        return False
    if c["denoise_to_zero"] or c["schedule"] == "edm" or c["eta"] == 0:
        return False
    if c["order"] == 3 and c["solver_type"] != "taylor":
        return False
    return c["order"] == 1 or not c["lower_order_final"] or c["steps"] >= 10


def _x0_fp64(mt, o, x, a, s):
    if mt == "noise":
        return (x - s * o) / a
    if mt == "x_start":
        return o
    if mt == "v":
        return a * x - s * o
    if mt == "score":
        return (x + s * s * o) / a
    return x - s * o                        # flow: x0 = x - t*v


def _kdiff(c, rig, s, x, draws):
    """The float64 k-diffusion loop of `c` on the product's grid, rig's network in float64, fed `draws`."""
    from dpm_solver_b200 import plan as P
    ns = rig.ns
    t_0 = 1. / ns.total_N if c["t_end"] is None else c["t_end"]
    t_T = ns.T if c["t_start"] is None else c["t_start"]
    ts = s.get_time_steps(c["skip_type"], t_T, t_0, c["steps"], "cpu")
    m = P.Marginals(ns, ts)
    al, ale, sg = (v.double().numpy() for v in (m.alpha, m.alpha_e, m.sigma))
    tin = rig.fn.get_model_input_time(ts).double().numpy()
    mt = c["model_type"]

    def denoise(xv, i):
        o = 0.1 * xv + ((tin[i] * 0.001) * 0.05 - 0.02)
        return _x0_fp64(mt, o, xv, ale[i], sg[i])
    return kdiff_sde(x.double().cpu().numpy(), denoise, al, sg, [z.double().numpy() for z in draws], c["eta"],
                     c["order"], c["solver_type"])


def oracle(c, device="cpu", seed=None):
    """{"y", "inter", "calls", "offset"} of the executor on `device` (the generator's offset after the run, None for a
    CPU generator), plus "pinned": "eta=0" or the k-diffusion distance when a pin was checked; {"error": exception}
    when the product refuses the configuration. An eta = 0 run draws nothing: it runs on the CPU (the numpy executor's
    ODE steps take CPU tensors) and its "offset" is None."""
    import dpm_solver_b200 as new
    seed = c["seed"] if seed is None else seed
    device = device if c["eta"] else "cpu"
    out = {}
    be = SdeOracle()
    with backend(be):
        rig = used = None
        try:
            rig = SdeRig(new, c, device)
            s = rig.solver()
            gen = rig.generator(seed)
            used = gen if isinstance(gen, torch.Generator) else default_generator(device)
            before = used.get_state()
            out["y"], out["inter"], out["calls"] = rig.sample(s, rig.x(), trace=True, gen=gen)
        except (ValueError, AssertionError) as e:
            # a refusal comes before any launch, network call or draw
            assert be.launch_count() == 0 and not be.draws and not getattr(rig, "trace_log", None), (c, e)
            assert used is None or torch.equal(used.get_state(), before), (c, e)
            return {"error": e}
        out["offset"] = used.get_offset() if rig.device.type == "cuda" else None
        out["draws"] = len(be.draws)
        if c["eta"] == 0:
            assert not be.draws and torch.equal(used.get_state(), before), c
            ode = SdeRig(new, dict(c, algo="dpmsolver++"), device)
            yo, io, co = _ode_run(ode)
            assert same_bits(out["y"], yo) and co == out["calls"], c
            assert len(io) == len(out["inter"]) and all(same_bits(a, b) for a, b in zip(io, out["inter"])), c
            out["pinned"] = "eta=0"
        else:
            assert len(be.draws) == c["steps"], (c, len(be.draws))
        if kdiff_expressible(c):
            want = _kdiff(c, rig, s, rig.x(), be.draws)
            err = max(float(np.abs(a.double().cpu().numpy() - b).max() / np.abs(b).max())
                      for a, b in zip(out["inter"], want))
            assert len(want) == len(out["inter"]) and err <= KDIFF_TOL, (c, err)
            out["pinned"] = err
    return out


def _ode_run(rig):
    """(y, intermediates, calls) of the rig's configuration as an ODE run (no eta, no generator)."""
    from gpu_configs import Rig
    return Rig.sample(rig, rig.solver(), rig.x(), trace=True)


# ---- the tally -------------------------------------------------------------------------------------------------------

def tally_static(c):
    """Entries that follow from a configuration the product accepts (also computed without a device)."""
    ps = per_sample(c)
    keys = ["schedule:" + ("vp" if c["schedule"] not in ("flow", "edm") else c["schedule"]), "order:%d" % c["order"],
            "solver_type:" + c["solver_type"], "eta:%g" % c["eta"], "generator:" + c["generator"],
            "skip:" + c["skip_type"], "guidance:" + ("rescale" if c["phi"] else c["guidance"]),
            "model:" + c["model_type"]]
    if c["feature"] != "plain":
        keys.append("guidance:" + c["feature"])
    if ps % 8:
        keys.append("step:element path")
    if c["thresholding"]:
        keys.append("thresholding")
        if c["feature"] == "tcfg":
            keys.append("tcfg:materialised")
    if c["state_dtype"]:
        keys.append("state:16-bit")
    if c["model_dtype"] and not c["state_dtype"]:
        keys.append("model:16-bit, state fp32")
    x_cl = c["x_channels_last"] and really_channels_last(dict(c, channels_last=True))
    if x_cl:
        keys.append("x:channels_last")
        if c["net_layout"] == "row":
            keys.append("layout change:row-major outputs of a channels_last state")
    if c["net_layout"] == "cl" and not c["x_channels_last"] and really_channels_last(c):
        keys.append("layout change:channels_last outputs of a row-major state")
    if c["denoise_to_zero"]:
        keys.append("d2z")
    if c["t_start"] is not None or c["t_end"] is not None:
        keys.append("t_start/t_end")
    return keys


REQUIRED = (["schedule:" + s for s in ("vp", "flow", "edm")] + ["order:%d" % o for o in (1, 2, 3)] +
            ["solver_type:dpmsolver", "solver_type:taylor"] + ["eta:%g" % e for e in ETAS] +
            ["generator:explicit", "generator:default"] +
            ["skip:" + k for k in ("time_uniform", "logSNR", "time_quadratic")] +
            ["guidance:" + g for g in ("none", "float", "tensor0", "per_sample", "rescale", "cfgzero", "tcfg", "fdg")] +
            ["step:element path", "thresholding", "tcfg:materialised", "state:16-bit", "model:16-bit, state fp32",
             "x:channels_last", "layout change:row-major outputs of a channels_last state",
             "layout change:channels_last outputs of a row-major state", "d2z", "t_start/t_end"])
REQUIRED_PINNED = ["pinned:eta=0", "pinned:kdiff"]
REQUIRED_REFUSED = ["refused:" + why for why in REFUSALS]
REQUIRED_ON_DEVICE = ["captured", "captured:eta>0", "second_stream", "frozen eta=0 step served", "rejected"]


def configurations(chunk):
    rng = random.Random(SEED + chunk)
    return [draw_sde(rng) for _ in range(PER_CHUNK)]
