"""Random CFG-Zero*, CFG++ and regional-guidance `sample()` configurations for the end-to-end tests on the device
(tests/test_gpu_guidance_random_configs.py) and their CPU side (tests/test_guidance_draws_vs_reference.py): the draw
(apg_configs.draw_apg's base, one feature per configuration), a `GuidanceRig` and the CPU oracle.

The base is draw_apg's: VP, flow and EDM schedules, 35 to 16384 elements per sample (some not multiples of 8), B from 1
to 4, a channels_last x_T, a network whose outputs keep their input's layout or are channels_last or row-major, 16-bit
state and model dtypes, inverse(), denoise_to_zero, t_start / t_end, skip types and lower_order_final. Then:
  * cfgzero: one scale from {1 (the bypass), 3.5, 7.5} or per-sample scales with rows at 1; cfg_zero_init_steps from
    {0, 1, 2, more than the run's evaluations}; DPM_Solver (every method) or UniPC; thresholding now and then.
  * cfgpp: DPM-Solver++ multistep of order 1 or 2, one scale from {0.2, 0.6, 1.0, 7.5} or per-sample scales; now and
    then a configuration CFG++ refuses (dpmsolver, order 3, singlestep, adaptive, UniPC, thresholding).
  * mask: K = 1..4 conditions, each with a mask of one of MASK_KINDS, held as fp32 (read in place when canonical),
    channels_last, bf16 or on the CPU (converted); values 0, negatives and quarters. UniPC is drawn now and then and
    must be refused.

The oracle of a configuration, on CPU tensors:
  * the product's host logic on the numpy executor `MaskOracle(exact=True)` (which is also the CFG++, CFG-Zero* and APG
    executor): y, every intermediate and the trace of network calls -- what the device must give bit for bit;
  * where the unmodified reference can express the configuration, the executor against it with as many network calls:
    cfgzero bit for bit through cfgzero_oracle.guided_net, cfgpp within CFGPP_TOL of cfgpp_oracle.cfgpp_fp64, mask bit
    for bit against test_cfg_mask.reference_composed;
  * a configuration the product refuses is {"error": exception}.
"""
import contextlib
import io
import random

import numpy as np
import torch

from apg_configs import APGRig, draw_apg, per_sample, reference_schedule
from cfg_mask_oracle import MaskOracle
from gpu_configs import backend, really_channels_last, rel_err, same_bits, sample_kwargs

FEATURES = ("cfgzero", "cfgpp", "mask")
BEYOND = 1000                 # a cfg_zero_init_steps above any run's number of evaluations: every evaluation is 0
CFGPP_TOL = 1e-5              # tests/test_cfg_pp.py's bound against the fp64 transcription
MASK_KINDS = ("hw", "11hw", "b1hw", "b111", "bchw", "chw", "bc11", "none")
MASK_FORMS = ("f32", "f32", "cl", "bf16", "cpu")
VP = ("sd", "ddpm_linear", "vp_linear")
CFGPP_REFUSALS =("dpmsolver", "order3", "singlestep", "adaptive", "unipc", "thresholding")
CHUNKS, PER_CHUNK, SEED = 6, 20, 9900     # the device test: 6 chunks of 20 configurations


def draw_guidance(rng):
    c = draw_apg(rng)
    c.update(apg_eta=None, apg_thr="off", apg_momentum=0.0, phi=0.0, tuning="auto")
    f = c["feature"] = rng.choice(FEATURES)
    B = c["B"]
    c["zero_init"], c["K"], c["masks"], c["cfgpp_refusal"] = 0, 0, None, None
    if c["schedule"] in ("flow", "edm") and rng.random() < {"cfgzero": 0.25, "cfgpp": 0.25, "mask": 0.5}[f]:
        c.update(schedule=rng.choice(VP), model_type=rng.choice(["noise", "x_start", "v", "score"]))
    if f in ("cfgzero", "cfgpp"):
        ones = [1.0, 3.5, 7.5] if f == "cfgzero" else [0.2, 0.6, 1.0, 7.5]
        if rng.random() < 0.4:
            rows = [rng.choice([7.5, 1.0, 3.5, 0.6]) for _ in range(B)]
            if B > 1 and 1.0 not in rows:
                rows[rng.randrange(B)] = 1.0
            c.update(guidance="per_sample", cfg=None, scales=rows)
        else:
            c.update(guidance="float", cfg=rng.choice(ones), scales=None)
    if f == "cfgzero":
        c["zero_init"] = rng.choice([0, 0, 1, 2, BEYOND])
        if c["sampler"] == "unipc" and c["guidance"] == "per_sample" and rng.random() < 0.7:
            c.update(guidance="float", cfg=7.5, scales=None)             # (UniPC refuses per-sample scales)
        if c["sampler"] == "dpm" and c["method"] == "adaptive" and c["zero_init"] and rng.random() < 0.6:
            c["zero_init"] = 0                                           # (refused; keep most adaptive draws)
    elif f == "cfgpp":
        c.update(sampler="dpm", method="multistep", order=rng.choice([1, 2]), algo="dpmsolver++", thresholding=False,
                 reference_rounding=False, steps=max(c["steps"], 3))
        if rng.random() < 0.15:
            why = c["cfgpp_refusal"] = rng.choice(CFGPP_REFUSALS)
            c.update({"dpmsolver": dict(algo="dpmsolver"), "order3": dict(order=3), "singlestep": dict(method="singlestep"),
                      "adaptive": dict(method="adaptive", order=2, atol=0.0078, rtol=0.05, inverse=False),
                      "unipc": dict(sampler="unipc", variant="bh2", use_corrector=False),
                      "thresholding": dict(thresholding=True)}[why])
    else:
        if len(c["shape"]) != 3:
            c["shape"] = rng.choice([(4, 64, 64), (3, 5, 7), (3, 8, 10)])
            c["net_layout"], c["x_channels_last"] = "keep", False
            c["channels_last"] = False
        if c["sampler"] == "unipc" and rng.random() < 0.85:
            c["sampler"] = "dpm"
        c["steps"] = max(c["steps"], c["order"])
        K = c["K"] = rng.randint(1, 4)
        c["masks"] = [(rng.choice(MASK_KINDS), rng.choice(MASK_FORMS)) for _ in range(K)]
        c.update(guidance="multi", cfg=None, scales=[rng.choice([7.5, -2.0, 0.0, 1.5, 3.0, 1.0]) for _ in range(K)])
    return c


def mask_shape(kind, B, shape):
    C, H, W = shape
    return {"hw": (H, W), "11hw": (1, 1, H, W), "b1hw": (B, 1, H, W), "b111": (B, 1, 1, 1), "bchw": (B, C, H, W),
            "chw": (C, H, W), "bc11": (B, C, 1, 1)}[kind]


def make_masks(c, device):
    """The configuration's masks on `device` ("cpu" masks stay on the CPU): quarters in [-1, 2], so 0, negatives and
    non-integers."""
    out = []
    for k, (kind, form) in enumerate(c["masks"]):
        if kind == "none":
            out.append(None)
            continue
        g = torch.Generator().manual_seed(c["seed"] + 101 * (k + 1))
        v = torch.randint(-4, 9, mask_shape(kind, c["B"], c["shape"]), generator=g).float() * 0.25
        if form == "bf16":
            v = v.to(torch.bfloat16)
        if form != "cpu":
            v = v.to(device)
        if form == "cl" and v.dim() == 4:
            v = v.contiguous(memory_format=torch.channels_last)
        out.append(v)
    return out


class GuidanceRig(APGRig):
    """APGRig with CFG-Zero*, CFG++ or regional guidance in model_wrapper. `masks` replaces the drawn masks."""

    def __init__(self, mod, c, device="cpu", masks=None):
        super().__init__(mod, dict(c, guidance="none"), device)
        self.c = c
        B, dev = c["B"], self.device
        kw = dict(model_type=c["model_type"], guidance_type="classifier-free",
                  unconditional_condition=torch.zeros(B, 1, device=dev))
        self.masks = None
        if c["feature"] == "mask":
            self.masks = make_masks(c, dev) if masks is None else masks
            cond = [torch.full((B, 1), float(k + 1), device=dev) for k in range(c["K"])]
            self.fn = mod.model_wrapper(self.net, self.ns, condition=cond, guidance_scale=list(c["scales"]),
                                        guidance_mask=self.masks, **kw)
            return
        scale = c["cfg"]
        if c["guidance"] == "per_sample":
            scale = torch.tensor(c["scales"], dtype=torch.float32, device=dev)
        self.scale = scale
        if c["feature"] == "cfgzero":
            kw.update(cfg_zero_star=True, cfg_zero_init_steps=c["zero_init"])
        else:
            kw["cfg_pp"] = True
        self.fn = mod.model_wrapper(self.net, self.ns, condition=torch.ones(B, 1, device=dev), guidance_scale=scale,
                                    **kw)


def refused(c):
    """Whether the product must refuse `c` with a ValueError before any launch."""
    if c["schedule"] == "flow" and c["model_type"] in ("v", "score"):
        return True
    if c["reference_rounding"]:
        return True          # (UniPC refuses it, and DPM_Solver does with each of the three features)
    unipc = c["sampler"] == "unipc"
    if unipc and c["steps"] < c["order"]:
        return True
    f = c["feature"]
    if f == "cfgzero":
        if unipc:
            return c["guidance"] == "per_sample" and c["B"] > 1
        return c["method"] == "adaptive" and c["zero_init"] > 0
    if f == "cfgpp":
        return (unipc or c["algo"] != "dpmsolver++" or c["method"] != "multistep" or c["order"] not in (1, 2)
                or c["thresholding"])
    return unipc


# ---- the reference ---------------------------------------------------------------------------------------------------

def _fp32(c):
    return c["state_dtype"] is None and c["model_dtype"] is None


def reference_expressible(c):
    """cfgzero: fp32 DPM_Solver, not adaptive, a network the reference's wrappers take on its schedule; cfgpp: fp32, a
    network with a closed-form x0, no denoise_to_zero; mask: fp32 DPM_Solver on a VP schedule, not adaptive. Never
    inverse()."""
    if refused(c) or not _fp32(c) or c["inverse"] or c["sampler"] != "dpm" or c["method"] == "adaptive":
        return False
    sched, mt = c["schedule"], c["model_type"]
    if c["feature"] == "cfgzero":
        return mt == sched if sched in ("flow", "edm") else mt in ("noise", "x_start", "v", "score")
    if c["feature"] == "cfgpp":
        return mt in ("noise", "x_start", "v", "score", "flow") and sched != "edm" and not c["denoise_to_zero"]
    return sched not in ("flow", "edm") and mt in ("noise", "x_start", "v", "score")


def _reference_cfgzero(c, rig, x):
    from cfgzero_oracle import guided_net
    from gpu_configs import reference
    ref = reference()
    B = c["B"]
    w = c["cfg"] if c["guidance"] == "float" else torch.tensor(c["scales"], dtype=torch.float32)
    rns = reference_schedule(c)
    g = guided_net(rig.net, torch.zeros(B, 1), torch.ones(B, 1), w, c["zero_init"])
    thr = c["thresholding"]
    if c["schedule"] in ("flow", "edm"):
        from edm_oracle import reference_solver as edm_solver
        from flow_oracle import reference_solver as flow_solver
        s = (flow_solver if c["schedule"] == "flow" else edm_solver)(g, rns, c["algo"], thr)
    else:
        s = ref.DPM_Solver(ref.model_wrapper(g, rns, model_type=c["model_type"]), rns, algorithm_type=c["algo"],
                           correcting_x0_fn="dynamic_thresholding" if thr else None)
    s.thresholding_max_val, s.dynamic_thresholding_ratio = c["max_val"], c["ratio"]
    rig.calls = []
    with contextlib.redirect_stdout(io.StringIO()):
        return s.sample(x, **sample_kwargs(c)), len(rig.calls)


def _reference_mask(c, rig, x):
    from test_cfg_mask import reference_composed
    n = [0]
    ref, rns, composed = reference_composed(c["model_type"], c["K"], c["scales"], [None if m is None else m.cpu()
                                                                                    for m in rig.masks],
                                            batch=c["B"], net=rig.net, sched=c["schedule"])

    def counted(xx, t):
        n[0] += 1
        return composed(xx, t)
    s = ref.DPM_Solver(counted, rns, algorithm_type=c["algo"],
                       correcting_x0_fn="dynamic_thresholding" if c["thresholding"] else None)
    s.thresholding_max_val, s.dynamic_thresholding_ratio = c["max_val"], c["ratio"]
    with contextlib.redirect_stdout(io.StringIO()):
        return s.sample(x, **sample_kwargs(c)), n[0]


def _reference_cfgpp(c, rig, x):
    """cfgpp_fp64 on the product's grid and fp32 marginals, the network's halves converted to x0 in fp64."""
    import dpm_solver_b200 as new
    from cfgpp_oracle import cfgpp_fp64
    from dpm_solver_b200 import plan as P
    ns, B, mt = rig.ns, c["B"], c["model_type"]
    s = new.DPM_Solver(rig.fn, ns)
    t_0 = 1. / ns.total_N if c["t_end"] is None else c["t_end"]
    t_T = ns.T if c["t_start"] is None else c["t_start"]
    ts = s.get_time_steps(c["skip_type"], t_T, t_0, c["steps"], "cpu")
    m = P.Marginals(ns, ts)
    lam, al, sg = (v.double().numpy() for v in (m.lam, m.alpha, m.sigma))
    tin = rig.fn.get_model_input_time(ts)
    w = np.float64(c["cfg"]) if c["guidance"] == "float" else \
        np.array(c["scales"], np.float64).reshape((B,) + (1,) * len(c["shape"]))
    n = [0]

    def x0(out, xx, i):
        out = out.astype(np.float64)
        if mt == "noise":
            return (xx - sg[i] * out) / al[i]
        if mt == "x_start":
            return out
        if mt == "v":
            return al[i] * xx - sg[i] * out
        if mt == "score":
            return (xx + sg[i] ** 2 * out) / al[i]
        return xx - sg[i] * out          # flow: x0 = x - t*v

    def pair(xx, i):
        n[0] += 1
        xt = torch.from_numpy(xx)
        t = tin[i].expand(B)
        cc, uu = rig.net(xt, t, torch.ones(B, 1)).double().numpy(), rig.net(xt, t, torch.zeros(B, 1)).double().numpy()
        U, C = x0(uu, xx, i), x0(cc, xx, i)
        return U + w * (C - U), U
    y = cfgpp_fp64(pair, lam, al, x.double().numpy(), c["order"], c["solver_type"], c["lower_order_final"])
    return torch.from_numpy(y), n[0]


def reference_run(c, rig):
    """(y, number of evaluations) of the reference form of `c` on rig's network."""
    x = rig.x()
    return {"cfgzero": _reference_cfgzero, "cfgpp": _reference_cfgpp, "mask": _reference_mask}[c["feature"]](c, rig, x)


def cpu_oracle(c):
    """{"y", "inter", "calls"} of the exact executor, plus "pinned" (the distance to the reference) when it was
    compared; {"error": exception} when the product refuses the configuration."""
    import dpm_solver_b200 as new
    out = {}
    with backend(MaskOracle(exact=True)):
        try:
            rig = GuidanceRig(new, c)
            out["y"], out["inter"], out["calls"] = rig.sample(rig.solver(), rig.x(), trace=True)
        except (ValueError, AssertionError) as e:
            return {"error": e}
        if reference_expressible(c):
            yr, n = reference_run(c, GuidanceRig(new, c))
            assert len(out["calls"]) == n, (c, len(out["calls"]), n)
            if c["feature"] == "cfgpp":
                out["pinned"] = rel_err(out["y"], yr)
                assert out["pinned"] <= CFGPP_TOL, (c, out["pinned"])
            else:
                assert same_bits(out["y"], yr), (c, rel_err(out["y"], yr))
                out["pinned"] = 0.0
    return out


# ---- the tally -------------------------------------------------------------------------------------------------------

def _is_cl(t):
    return t.dim() == 4 and not t.is_contiguous() and t.is_contiguous(memory_format=torch.channels_last)


def tally_static(c):
    """Entries that follow from a configuration the product accepts (also computed without a device)."""
    f = c["feature"]
    ps = per_sample(c)
    keys = ["feature:" + f, "schedule:" + ("vp" if c["schedule"] not in ("flow", "edm") else c["schedule"]),
            "sampler:" + c["sampler"]]
    if ps % 8:
        keys.append("step:scalar")
    if c["thresholding"]:
        keys.append("quantile:pipeline" if ps >= 8192 else "quantile:cluster")
    if c["guidance"] == "per_sample" and c["B"] > 1 and 1.0 in c["scales"]:
        keys.append("bypassed row")
    if c["state_dtype"]:
        keys.append("state:16-bit")
    x_cl = c["x_channels_last"] and really_channels_last(dict(c, channels_last=True))
    if x_cl:
        keys.append("x:channels_last")
        if c["net_layout"] == "row":
            keys.append("layout change:row-major outputs of a channels_last state")
    if c["net_layout"] == "cl" and not c["x_channels_last"] and really_channels_last(c):
        keys.append("layout change:channels_last outputs of a row-major state")
    if c["sampler"] == "dpm":
        keys.append("method:" + c["method"])
    if c["inverse"]:
        keys.append("inverse")
    if c["denoise_to_zero"]:
        keys.append("d2z")
    if c["t_start"] is not None or c["t_end"] is not None:
        keys.append("t_start/t_end")
    if f == "cfgzero":
        keys.append("zero-init:" + {0: "none", BEYOND: "all"}.get(c["zero_init"], "partial"))
    elif f == "cfgpp":
        keys.append("cfgpp:order%d" % c["order"])
        if c["cfg"] == 1.0:
            keys.append("cfgpp:scale 1")
    else:
        keys.append("mask:K=%d" % c["K"])
        for (kind, form), m in zip(c["masks"], make_masks(c, "cpu")):
            keys.append("mask:" + kind)
            if m is not None and (form in ("bf16", "cpu") or _is_cl(m)):
                keys.append("mask:converted")
            if m is not None and x_cl and kind not in ("b111", "bc11"):
                keys.append("mask:channels_last element map")
    return keys


REQUIRED = (["feature:" + f for f in FEATURES] + ["schedule:vp", "schedule:flow", "schedule:edm", "sampler:dpm",
                                                  "sampler:unipc"] +
            ["zero-init:none", "zero-init:partial", "zero-init:all", "cfgpp:order1", "cfgpp:order2", "cfgpp:scale 1",
             "bypassed row"] +
            ["mask:" + k for k in MASK_KINDS] + ["mask:K=%d" % k for k in (1, 2, 3, 4)] +
            ["mask:converted", "mask:channels_last element map", "step:scalar", "quantile:pipeline",
             "quantile:cluster", "state:16-bit", "x:channels_last",
             "layout change:row-major outputs of a channels_last state",
             "layout change:channels_last outputs of a row-major state"] +
            ["method:" + m for m in ("multistep", "singlestep", "singlestep_fixed", "adaptive")] +
            ["inverse", "d2z", "t_start/t_end"])
REQUIRED_ON_DEVICE = ["rejected", "captured", "captured:zero-init", "captured:rewritten-mask", "second_stream",
                      "pinned"]


def configurations(chunk):
    rng = random.Random(SEED + chunk)
    return [draw_guidance(rng) for _ in range(PER_CHUNK)]
