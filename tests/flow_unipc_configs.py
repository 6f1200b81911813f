"""Random flow-matching and UniPC `sample()` configurations for the end-to-end tests on the device
(tests/test_gpu_flow_unipc_random_configs.py, tests/test_unipc_reuse.py): the draw (gpu_configs.draw_gpu, extended),
a `FlowRig` that builds a flow or VP schedule and a DPM_Solver or UniPC on it, and the CPU oracle.

The oracle of a configuration, on CPU tensors:
  * the product's host logic on the numpy executor (`UniPCOracle`, which is also the flow executor): y, every
    intermediate and the trace of network calls, for every configuration;
  * a flow DPM_Solver configuration the unmodified reference can express (fp32 state and network, the guidance forms
    `flow_oracle.reference_model` writes, not the adaptive method) must come out of the executor bit for bit as
    `flow_oracle.reference_solver` (a velocity network) or the reference's own model_wrapper (noise, x_start) computes it;
  * UniPC bh2 of order <= 2 without the corrector, whose final orders are DPM-Solver's, in fp32 with at most one scale,
    must equal the reference's multistep DPM-Solver(++)(2M) to `UNIPC_2M_TOL` relative (the bound of
    tests/test_unipc.py), the trace of network calls exactly;
  * a configuration the product rejects (a `v` or `score` network on a flow schedule, `reference_rounding` there or with
    UniPC, per-sample scales, several conditions or the rescale with UniPC, steps < order) is {"error": exception}.
"""
import contextlib
import io
import random

import torch

import flow_oracle as F
from gpu_configs import DT, Rig, backend, draw_gpu, reference, rel_err, really_channels_last, same_bits, sample_kwargs
from unipc_oracle import UniPCOracle

SHIFTS = [1.0, 3.0, 1.15]
TIME_SCALES = [1000.0, 1.0]
UNIPC_2M_TOL = 1e-6
CHUNKS, PER_CHUNK, SEED = 6, 20, 9400     # the device test: 6 chunks of 20 configurations


def draw_flow_unipc(rng):
    """draw_gpu() on a flow schedule (shift, time_scale, a velocity, noise or x_start network; now and then a `v` or
    `score` one, which must be refused) or, for UniPC only, on draw_gpu's VP schedule; the sampler DPM_Solver (every
    method) or UniPC (variant, order 1-3, corrector, lower_order_final)."""
    c = draw_gpu(rng)
    c["sampler"] = "unipc" if rng.random() < 0.55 else "dpm"
    unipc = c["sampler"] == "unipc"
    if not unipc or rng.random() < 0.75:
        c.update(schedule="flow", shift=rng.choice(SHIFTS), time_scale=rng.choice(TIME_SCALES))
        c["model_type"] = rng.choice(["flow", "flow", "flow", "noise", "x_start"] if rng.random() < 0.95 else
                                     ["v", "score"])
    if c["algo"] == "dpmsolver++" and rng.random() < 0.2:     # (the pipeline quantile: >= 8192 per sample)
        c.update(thresholding=True, shape=(4, 64, 64), B=rng.choice([1, 2]))
        if c["guidance"] == "per_sample":
            c["scales"] = [rng.choice([7.5, 1.0, 0.0, -2.0, 3.5]) for _ in range(c["B"])]
    c["reference_rounding"] = rng.random() < 0.03
    if unipc:
        c.update(method="multistep", variant=rng.choice(["bh1", "bh2"]), order=rng.choice([1, 2, 3]),
                 use_corrector=rng.random() < 0.7)
        if rng.random() < 0.1:
            c["steps"] = rng.randint(1, 3)               # (below the order now and then: refused)
        if c["guidance"] in ("per_sample", "multi", "rescale") and rng.random() < 0.7:
            # (UniPC refuses those three; keep most UniPC draws runnable)
            c["guidance"] = rng.choice(["none", "float", "tensor0"])
            c["cfg"] = None if c["guidance"] == "none" else rng.choice([1.0, 3.5, 7.5])
            c["scales"], c["phi"] = None, 0.0
        if rng.random() < 0.35:                          # bh2, UniP-2 without the corrector: the reference's 2M
            c.update(variant="bh2", order=rng.choice([1, 2]), use_corrector=False, lower_order_final=False)
    return c


class FlowRig(Rig):
    """gpu_configs.Rig on the configuration's schedule (flow or VP), with a DPM_Solver or a UniPC as its solver."""

    def make_schedule(self):
        c = self.c
        if c["schedule"] != "flow":
            return super().make_schedule()
        return self.mod.NoiseScheduleFlow(shift=c["shift"], time_scale=c["time_scale"])

    def solver(self, **kw):
        c = self.c
        if c["sampler"] != "unipc":
            if c.get("reference_rounding"):
                kw["reference_rounding"] = True
            return super().solver(**kw)
        kw.setdefault("state_dtype", DT[c["state_dtype"]])
        s = self.mod.UniPC(self.fn, self.ns, algorithm_type=c["algo"], variant=c["variant"],
                           correcting_x0_fn="dynamic_thresholding" if c["thresholding"] else None,
                           thresholding_max_val=c["max_val"], dynamic_thresholding_ratio=c["ratio"], **kw)
        s.reference_rounding = bool(c.get("reference_rounding"))
        return s

    def kwargs(self):
        """The sampling arguments of the configuration (without return_intermediate)."""
        c = self.c
        if c["sampler"] != "unipc":
            return sample_kwargs(c)
        return dict(steps=c["steps"], order=c["order"], skip_type=c["skip_type"], lower_order_final=c["lower_order_final"],
                    denoise_to_zero=c["denoise_to_zero"], t_end=c["t_end"], t_start=c["t_start"],
                    use_corrector=c["use_corrector"])

    def sample(self, s, x, trace=False, **over):
        if self.c["sampler"] != "unipc":
            return super().sample(s, x, trace, **over)
        self.calls = [] if trace else None
        try:
            y, inter = s.sample(x, return_intermediate=True, **dict(self.kwargs(), **over))
            return y, inter, self.calls
        finally:
            self.calls = None


def refused(c):
    """Whether the product must refuse `c` with a ValueError before any launch."""
    if c["schedule"] == "flow" and c["model_type"] in ("v", "score") or c["reference_rounding"]:
        return True
    if c["guidance"] == "multi" and c["phi"]:
        return True                     # (model_wrapper: the rescale with several conditions)
    # (a one-element scale tensor, per_sample at B = 1, is one scale)
    per_sample = c["guidance"] == "per_sample" and c["B"] > 1
    return c["sampler"] == "unipc" and (per_sample or c["guidance"] == "multi" or bool(c["phi"])
                                        or c["steps"] < c["order"])


# ---- the references ----------------------------------------------------------------------------------------------
def _fp32(c):
    return c["state_dtype"] is None and c["model_dtype"] is None and not c.get("reference_rounding")


def flow_reference_expressible(c):
    """A flow DPM_Solver configuration the unmodified reference computes: fp32, every guidance form of
    flow_oracle.reference_model for a velocity network (a scale of 1 keeps its doubled batch there, not the
    reference wrapper's single call), one scale or none for a noise or x_start one (the reference's own wrapper)."""
    if c["sampler"] != "dpm" or c["schedule"] != "flow" or not _fp32(c) or c["method"] == "adaptive":
        return False
    g = c["guidance"]
    if c["model_type"] == "flow":
        if c["phi"] and g != "rescale":
            return False
        return g in ("none", "per_sample", "multi") or c["cfg"] != 1.0
    return c["model_type"] in ("noise", "x_start") and g in ("none", "float", "tensor0")


def unipc_is_2m(c):
    """UniPC configurations that are the reference's multistep DPM-Solver(++)(2M) (or DDIM) in exact arithmetic:
    bh2, order <= 2, no corrector, the same final orders (UniPC lowers them at any number of steps, DPM-Solver below
    10 steps only), fp32, one scale or none, and for a flow schedule a network the reference can be driven with."""
    if c["sampler"] != "unipc" or c["variant"] != "bh2" or c["order"] > 2 or c["use_corrector"]:
        return False
    if c["steps"] < c["order"] or not _fp32(c) or c["guidance"] not in ("none", "float", "tensor0"):
        return False
    if c["order"] == 2 and c["lower_order_final"] and c["steps"] >= 10:
        return False
    if c["schedule"] == "flow" and c["model_type"] == "flow" and c["cfg"] == 1.0:
        return False
    return c["schedule"] != "flow" or c["model_type"] in ("flow", "noise", "x_start")


def reference_flow_solver(c, rig):
    """The unmodified reference DPM_Solver on flow configuration `c`, calling `rig.net` (a product FlowRig on CPU: its
    network, not its schedule or wrapper), so that the trace lands in `rig.calls`."""
    ref = reference()
    rns = F.reference_schedule(c["shift"], c["time_scale"])
    B, g = c["B"], c["guidance"]
    uc = torch.zeros(B, 1)
    if c["model_type"] == "flow":
        kw = {}
        if g != "none":
            if g == "multi":
                conds, scales, kind = [torch.full((B, 1), float(k + 1)) for k in range(len(c["scales"]))], list(c["scales"]), "multi"
            elif g == "per_sample":
                conds, scales, kind = [torch.ones(B, 1)], list(c["scales"]), "per_sample"
            else:
                conds, scales, kind = [torch.ones(B, 1)], c["cfg"], "scalar"
            kw = dict(guidance=dict(uc=uc, conds=conds, scales=scales, kind=kind), phi=c["phi"])
        s = F.reference_solver(rig.net, rns, c["algo"], c["thresholding"], **kw)
    else:
        rns.schedule = "linear"          # the reference wrapper hands the network t itself: give it what ours gets
        net = lambda xx, tt, *cc: rig.net(xx, rns.input_time(tt), *cc)
        kw = dict(model_type=c["model_type"])
        if g != "none":
            kw.update(guidance_type="classifier-free", condition=torch.ones(B, 1), unconditional_condition=uc,
                      guidance_scale=c["cfg"])
        s = ref.DPM_Solver(ref.model_wrapper(net, rns, **kw), rns, algorithm_type=c["algo"],
                           correcting_x0_fn="dynamic_thresholding" if c["thresholding"] else None)
    s.thresholding_max_val, s.dynamic_thresholding_ratio = c["max_val"], c["ratio"]
    return s


def reference_run(c):
    """(y, intermediates, calls) of the reference on `c` (a UniPC configuration runs as multistep DPM-Solver)."""
    import dpm_solver_b200 as new
    if c["sampler"] == "unipc":
        c = dict(c, method="multistep", solver_type="dpmsolver")
    if c["schedule"] != "flow":
        rig = Rig(reference(), c)
        return rig.sample(rig.solver(), rig.x(), trace=True)
    rig = FlowRig(new, dict(c, sampler="dpm"))
    s = reference_flow_solver(c, rig)
    rig.calls = []
    with contextlib.redirect_stdout(io.StringIO()):
        y, inter = s.sample(rig.x(), return_intermediate=True, **sample_kwargs(c))
    return y, inter, rig.calls


def cpu_oracle(c):
    """{"y", "inter", "calls"} of the numpy executor, plus "pinned": "reference" (bit for bit) or "2M" (to
    UNIPC_2M_TOL) when a reference was compared; {"error": exception} when the product refuses the configuration."""
    import dpm_solver_b200 as new
    out = {}
    with backend(UniPCOracle()):
        try:
            rig = FlowRig(new, c)
            out["y"], out["inter"], out["calls"] = rig.sample(rig.solver(), rig.x(), trace=True)
        except (ValueError, AssertionError) as e:
            return {"error": e}
    if flow_reference_expressible(c):
        yr, ir, cr = reference_run(c)
        assert out["calls"] == cr, c
        assert same_bits(out["y"], yr) and len(out["inter"]) == len(ir), c
        assert all(same_bits(a, b) for a, b in zip(out["inter"], ir)), c
        out["pinned"] = "reference"
    elif unipc_is_2m(c):
        yr, ir, cr = reference_run(c)
        assert out["calls"] == cr, c
        assert len(out["inter"]) == len(ir), c
        for a, b in zip([out["y"]] + out["inter"], [yr] + ir):
            assert rel_err(a, b) <= UNIPC_2M_TOL, (c, rel_err(a, b))
        out["pinned"] = "2M"
    return out


# ---- the tally -----------------------------------------------------------------------------------------------------
def tally_static(c):
    """Entries that follow from a configuration the product accepts (also computed without a device)."""
    sampler = c["sampler"]
    keys = ["sampler:" + sampler]
    if c["schedule"] == "flow":
        keys += ["shift:%g" % c["shift"], "time_scale:%g" % c["time_scale"], "flow_model:" + c["model_type"],
                 "flow:" + sampler]
    else:
        keys.append("vp:" + sampler)
    if sampler == "unipc":
        keys += ["unipc:" + c["variant"], "unipc:order%d" % c["order"],
                 "unipc:corrector" if c["use_corrector"] else "unipc:no_corrector"]
        if c["lower_order_final"]:
            keys.append("unipc:lower_order_final")
        if c["state_dtype"] is None and c["model_dtype"] == "bf16":
            keys.append("unipc:bf16_net_fp32_state")
        if really_channels_last(c):
            keys.append("unipc:channels_last")
    else:
        keys.append("method:" + c["method"])
    if c["thresholding"]:
        n = 1
        for d in c["shape"]:
            n *= d
        keys.append(("quantile:pipeline:" if n >= 8192 else "quantile:cluster:") + sampler)
    if c["tuning"] == "tma":
        keys.append("tuning:tma")
    if c["state_dtype"]:
        keys.append("state:16-bit")
    if c["denoise_to_zero"]:
        keys.append("d2z")
    if c["t_start"] is not None or c["t_end"] is not None:
        keys.append("t_start/t_end")
    return keys


REQUIRED = (["shift:%g" % s for s in SHIFTS] + ["time_scale:%g" % s for s in TIME_SCALES] +
            ["flow_model:" + m for m in ("flow", "noise", "x_start")] + ["flow:dpm", "flow:unipc", "vp:unipc"] +
            ["unipc:bh1", "unipc:bh2", "unipc:order1", "unipc:order2", "unipc:order3", "unipc:corrector",
             "unipc:no_corrector", "unipc:lower_order_final", "unipc:bf16_net_fp32_state", "unipc:channels_last"] +
            ["quantile:%s:%s" % (q, s) for q in ("pipeline", "cluster") for s in ("dpm", "unipc")] +
            ["tuning:tma", "state:16-bit", "d2z", "t_start/t_end", "method:adaptive", "method:singlestep"])
REQUIRED_PINNED = ["pinned:reference", "pinned:2M"]
REQUIRED_ON_DEVICE = ["rejected", "captured", "second_stream"]


def configurations(chunk):
    """The configurations of one chunk of the device test."""
    rng = random.Random(SEED + chunk)
    return [draw_flow_unipc(rng) for _ in range(PER_CHUNK)]
