"""Random CFG-Zero*, CFG++, regional-guidance, TCFG, frequency-decoupled-guidance and Perp-Neg `sample()` configurations
for the end-to-end tests on the device (tests/test_gpu_guidance_random_configs.py) and their CPU side
(tests/test_guidance_draws_vs_reference.py): the draw (apg_configs.draw_apg's base, one feature per configuration), a
`GuidanceRig` and the CPU oracle.

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
  * tcfg: one scale from {1 (the bypass), 3.5, 7.5}, a one-element tensor scale, or per-sample scales with rows at 1;
    DPM_Solver (every method) or UniPC; thresholding now and then (both materialise g in fp32 before the step).
  * fdg: planes that reach each CTA shape of k_fdg_guided, its shared-memory opt-in and its scalar loads (FDG_PLANES),
    or the base's shape; `levels` from what the plane admits, and now and then one level more, which the size rule
    refuses; the scales as N floats, N one-element tensors, a 1-D tensor, an fp32 [B, N] tensor read in place, a bf16
    or CPU [B, N] tensor (converted), or a [B + 1, N] tensor (refused); now and then equal scales, whose run must be
    the N == 1 run.
  * perp: K = 2..4 conditions with scales from PERP_SCALES (negatives, 0 and 1), now and then a sample whose first
    condition is the unconditional one (||d_1|| = 0: its word is s_1); DPM_Solver (every method); now and then a
    configuration Perp-Neg refuses (PERP_REFUSALS: per-sample scales, a guidance_mask, UniPC, a single condition,
    reference_rounding).

The oracle of a configuration, on CPU tensors:
  * the product's host logic on the numpy executor -- `MaskOracle(exact=True)` (which is also the CFG++, CFG-Zero* and
    APG executor), for tcfg and fdg `FDGOracle()` (TCFG's words in the device's summation order), for perp
    `PerpNegOracle(exact=True)` (the words in the device's summation order): y, every intermediate and the trace of
    network calls -- what the device must give bit for bit;
  * where the unmodified reference can express the configuration, the executor against it with as many network calls:
    cfgzero, tcfg and fdg bit for bit through cfgzero_oracle / tcfg_oracle / fdg_oracle.guided_net behind a
    guidance_type="uncond" wrapper, cfgpp within CFGPP_TOL of cfgpp_oracle.cfgpp_fp64 (plus, for an x_start network,
    the rounding bound of its x0 conversion: _reference_cfgpp), mask bit for bit against
    test_cfg_mask.reference_composed, perp bit for bit through perpneg_oracle.guided_net behind a
    guidance_type="uncond" wrapper (a noise network) or test_perp_neg.reference_composed (the other model types);
  * a configuration the product refuses is {"error": exception}.
"""
import contextlib
import io
import random

import numpy as np
import torch

from apg_configs import APGRig, draw_apg, per_sample, reference_schedule
from cfg_mask_oracle import MaskOracle
from fdg_oracle import FDGOracle
from gpu_configs import backend, really_channels_last, rel_err, same_bits, sample_kwargs
from perpneg_oracle import PerpNegOracle

FEATURES = ("cfgzero", "cfgpp", "mask", "tcfg", "fdg", "perp")
BEYOND = 1000                 # a cfg_zero_init_steps above any run's number of evaluations: every evaluation is 0
CFGPP_TOL = 1e-5              # tests/test_cfg_pp.py's bound against the fp64 transcription
XSTART_ROUNDING = 3           # x_start under CFG++: multiples of what its fp32 x0 conversion alone moves a run
MASK_KINDS = ("hw", "11hw", "b1hw", "b111", "bchw", "chw", "bc11", "none")
MASK_FORMS = ("f32", "f32", "cl", "bf16", "cpu")
VP = ("sd", "ddpm_linear", "vp_linear")
CFGPP_REFUSALS =("dpmsolver", "order3", "singlestep", "adaptive", "unipc", "thresholding")
# k_fdg_guided's paths: 64 x 64 (CTA shape 0, 5 levels), 72 x 64 (shape 1), 64 x 128 (shape 1 past 48 KiB of shared
# memory), 126 x 130 (shape 2, H*W % 8 != 0: scalar loads), 6 x 6 (the smallest plane with 2 levels), 24 x 40
FDG_PLANES = [(4, 64, 64), (3, 72, 64), (2, 64, 128), (1, 126, 130), (2, 6, 6), (3, 24, 40)]
FDG_FORMS = ("floats", "listed", "vec", "rows", "rows", "bf16", "cpu")     # (+ "bad_rows" now and then: refused)
FDG_VALUES = [7.0, 3.5, 1.5, 1.0, 0.0, -1.0, 10.0, 2.5]                  # (exact in bf16)
PERP_SCALES = [7.5, 4.0, 1.0, 0.0, -1.0, -2.5, -0.5]
PERP_REFUSALS = ("per_sample", "mask", "unipc", "single", "rr")
CHUNKS, PER_CHUNK, SEED = 12, 22, 9900    # the device test: 12 chunks of 22 configurations


def draw_guidance(rng):
    c = draw_apg(rng)
    c.update(apg_eta=None, apg_thr="off", apg_momentum=0.0, phi=0.0, tuning="auto")
    f = c["feature"] = rng.choice(FEATURES)
    B = c["B"]
    c["zero_init"], c["K"], c["masks"], c["cfgpp_refusal"] = 0, 0, None, None
    c["fdg_levels"], c["fdg_form"], c["fdg_w"], c["fdg_equal"] = 0, None, None, False
    c["perp_refusal"], c["perp_d1_zero"] = None, None
    if c["schedule"] in ("flow", "edm") and rng.random() < {"cfgzero": 0.25, "cfgpp": 0.25, "mask": 0.5, "tcfg": 0.25,
                                                             "fdg": 0.25, "perp": 0.5}[f]:
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
    elif f == "tcfg":
        g = rng.random()
        if g < 0.35:
            rows = [rng.choice([7.5, 1.0, 3.5]) for _ in range(B)]
            if B > 1 and 1.0 not in rows:
                rows[rng.randrange(B)] = 1.0
            c.update(guidance="per_sample", cfg=None, scales=rows)
        elif g < 0.55:
            c.update(guidance="tensor0", cfg=rng.choice([1.0, 3.5, 7.5]), scales=None)
        else:
            c.update(guidance="float", cfg=rng.choice([1.0, 3.5, 7.5]), scales=None)
        if c["sampler"] == "unipc" and c["guidance"] == "per_sample" and rng.random() < 0.7:
            c.update(guidance="float", cfg=7.5, scales=None)             # (UniPC refuses per-sample scales)
        if c["algo"] == "dpmsolver++" and rng.random() < 0.15:
            c["thresholding"] = True
    elif f == "fdg":
        draw_fdg(rng, c)
    elif f == "perp":
        draw_perp(rng, c)
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


def draw_perp(rng, c):
    """The perp part of a draw: K, the scales, a sample with ||d_1|| = 0 now and then, a refusal now and then."""
    B = c["B"]
    if c["sampler"] == "unipc":
        c["sampler"] = "dpm"
    c["steps"] = max(c["steps"], c["order"])
    K = c["K"] = rng.randint(2, 4)
    c.update(guidance="perp", cfg=None, scales=[rng.choice(PERP_SCALES) for _ in range(K)])
    if rng.random() < 0.25:
        c["perp_d1_zero"] = rng.randrange(B)
    if rng.random() < 0.25:
        why = c["perp_refusal"] = rng.choice(PERP_REFUSALS)
        if why == "unipc":
            c.update(sampler="unipc", variant="bh2", use_corrector=False, method="multistep", inverse=False)
        elif why == "single":
            c.update(K=1, scales=c["scales"][:1])
        elif why == "rr":
            c["reference_rounding"] = True


def perp_refusal_reached(c):
    """Whether Perp-Neg's own refusal decides a perp draw that carries one: the same draw without it (the single
    condition, UniPC or reference_rounding undone) is one the product accepts, so no other check can refuse it first."""
    if c["feature"] != "perp" or c["perp_refusal"] is None:
        return False
    undone = dict(c, perp_refusal=None, K=max(c["K"], 2), scales=c["scales"] + [1.0] * (2 - len(c["scales"])))
    if c["perp_refusal"] == "unipc":
        undone["sampler"] = "dpm"
    if c["perp_refusal"] == "rr":
        undone["reference_rounding"] = False
    return not refused(undone)


def perp_conditions(c, device):
    """The K conditions [B, 1]: k + 1 for condition k, except 0 (the unconditional one) for condition 1 of sample
    c["perp_d1_zero"]."""
    cond = [torch.full((c["B"], 1), float(k + 1), device=device) for k in range(c["K"])]
    if c["perp_d1_zero"] is not None:
        cond[0][c["perp_d1_zero"]] = 0.0
    return cond


def perp_net(base):
    """`base` (APGRig's network, whose conditional differences are all parallel) plus (c*c/100)*y*y with y = x clamped
    to [-2, 2], a bounded condition term nonlinear in x: the differences d_k of distinct conditions are then not parallel, and Perp-Neg's perpendicular parts
    do not vanish. A condition of 0 adds nothing (||d_1|| = 0 stays exact). Exact IEEE products and sums, in the
    output's dtype and layout."""
    def net(xx, tt, cc=None):
        o = base(xx, tt, cc)
        if cc is None:
            return o
        one = (-1,) + (1,) * (xx.dim() - 1)
        y = xx.float().clamp(-2.0, 2.0)
        r = (o.float() + ((0.01 * cc.reshape(one)) * cc.reshape(one)) * (y * y)).to(o.dtype)
        cl = o.dim() == 4 and not o.is_contiguous() and o.is_contiguous(memory_format=torch.channels_last)
        return r.contiguous(memory_format=torch.channels_last) if cl else r.contiguous()
    return net


def fdg_max_levels(shape):
    """The most levels the size rule admits for the plane of `shape` (H and W divisible by 2^(levels-1), quotients of
    at least 3, at most 5 levels)."""
    H, W = shape[-2:]
    L = 1
    while L < 5 and H % (2 << (L - 1)) == 0 and W % (2 << (L - 1)) == 0 and H >> L >= 3 and W >> L >= 3:
        L += 1
    return L


def draw_fdg(rng, c):
    """The fdg part of a draw: the plane, the layouts on it, the levels and the scales."""
    if not c["thresholding"] or rng.random() < 0.5:
        c["shape"] = rng.choice(FDG_PLANES + [(2, 3, 6, 4), c["shape"]])
    c["steps"] = min(c["steps"], 12)
    three = len(c["shape"]) == 3
    c["x_channels_last"] = three and rng.random() < 0.3
    c["net_layout"] = rng.choice(["keep", "keep", "cl", "row"]) if three else "keep"
    c["channels_last"] = c["net_layout"] == "cl"
    c["x2_channels_last"] = three and not c["channels_last"] and rng.random() < 0.15
    c.update(guidance="fdg", cfg=None, scales=None)
    mx = fdg_max_levels(c["shape"])
    L = c["fdg_levels"] = mx + 1 if rng.random() < 0.1 else rng.choice([1, mx, mx] + list(range(1, mx + 1)))
    c["fdg_form"] = "bad_rows" if rng.random() < 0.05 else rng.choice(FDG_FORMS)
    c["fdg_equal"] = rng.random() < 0.15
    rows = []
    for _ in range(c["B"] if c["fdg_form"] not in ("floats", "listed", "vec") else 1):
        rows.append([rng.choice(FDG_VALUES)] * L if c["fdg_equal"] else [rng.choice(FDG_VALUES) for _ in range(L)])
    c["fdg_w"] = rows * c["B"] if len(rows) == 1 else rows


def make_fdg_scales(c, device):
    """The configuration's fdg_scales in its form: N floats, N one-element tensors, a 1-D tensor, an fp32 [B, N]
    tensor on `device` (read in place there), a bf16 one on `device` or an fp32 one on the CPU (both converted), or an
    fp32 [B + 1, N] tensor."""
    rows, form = c["fdg_w"], c["fdg_form"]
    if form == "floats":
        return list(rows[0])
    if form == "listed":
        return [torch.tensor([v], device=device) for v in rows[0]]
    if form == "vec":
        return torch.tensor(rows[0], device=device)
    if form == "bad_rows":
        rows = rows + rows[:1]
    t = torch.tensor(rows, dtype=torch.float32)
    return t if form == "cpu" else t.to(device=device, dtype=torch.bfloat16 if form == "bf16" else torch.float32)


def fdg_values(c):
    """The scales as the kernel reads them: N python floats (the shared forms) or an fp32 [B, N] CPU tensor."""
    if c["fdg_form"] in ("floats", "listed", "vec"):
        return list(c["fdg_w"][0])
    return torch.tensor(c["fdg_w"], dtype=torch.float32)


def executor(c):
    """The numpy executor of `c`: FDGOracle (which also runs TCFG) for tcfg and fdg, PerpNegOracle(exact=True) for perp,
    MaskOracle(exact=True) else."""
    if c["feature"] == "perp":
        return PerpNegOracle(exact=True)
    return FDGOracle() if c["feature"] in ("tcfg", "fdg") else MaskOracle(exact=True)


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
    """APGRig with CFG-Zero*, CFG++, regional guidance, TCFG, frequency-decoupled guidance or Perp-Neg in model_wrapper.
    `masks` replaces the drawn masks, `fdg` the drawn fdg_scales, `scales` the drawn Perp-Neg scales."""

    def __init__(self, mod, c, device="cpu", masks=None, fdg=None, scales=None):
        super().__init__(mod, dict(c, guidance="none"), device)
        self.c = c
        B, dev = c["B"], self.device
        kw = dict(model_type=c["model_type"], guidance_type="classifier-free",
                  unconditional_condition=torch.zeros(B, 1, device=dev))
        self.masks = self.fdg = None
        if c["feature"] == "fdg":
            self.fdg = make_fdg_scales(c, dev) if fdg is None else fdg
            self.fn = mod.model_wrapper(self.net, self.ns, condition=torch.ones(B, 1, device=dev), fdg_scales=self.fdg,
                                        **kw)
            return
        if c["feature"] == "perp":
            why = c["perp_refusal"]
            scale = list(c["scales"] if scales is None else scales)
            if why == "per_sample":
                scale = torch.tensor([scale] * B, dtype=torch.float32, device=dev).T.contiguous()    # [K, B]
            if why == "mask":
                kw["guidance_mask"] = [torch.ones(B, 1, 1, 1, device=dev)] + [None] * (c["K"] - 1)
            self.net = perp_net(self.net)
            self.fn = mod.model_wrapper(self.net, self.ns, condition=perp_conditions(c, dev), guidance_scale=scale,
                                        perp_neg=True, **kw)
            return
        if c["feature"] == "mask":
            self.masks = make_masks(c, dev) if masks is None else masks
            cond = [torch.full((B, 1), float(k + 1), device=dev) for k in range(c["K"])]
            self.fn = mod.model_wrapper(self.net, self.ns, condition=cond, guidance_scale=list(c["scales"]),
                                        guidance_mask=self.masks, **kw)
            return
        scale = c["cfg"]
        if c["guidance"] == "per_sample":
            scale = torch.tensor(c["scales"], dtype=torch.float32, device=dev)
        elif c["guidance"] == "tensor0":
            scale = torch.tensor(c["cfg"])
        self.scale = scale
        if c["feature"] == "cfgzero":
            kw.update(cfg_zero_star=True, cfg_zero_init_steps=c["zero_init"])
        elif c["feature"] == "tcfg":
            kw["tcfg"] = True
        else:
            kw["cfg_pp"] = True
        self.fn = mod.model_wrapper(self.net, self.ns, condition=torch.ones(B, 1, device=dev), guidance_scale=scale,
                                    **kw)


def refused(c):
    """Whether the product must refuse `c` with a ValueError before any launch."""
    if c["schedule"] == "flow" and c["model_type"] in ("v", "score"):
        return True
    if c["reference_rounding"]:
        return True          # (UniPC refuses it, and DPM_Solver does with each of the five features)
    unipc = c["sampler"] == "unipc"
    if unipc and c["steps"] < c["order"]:
        return True
    f = c["feature"]
    if f == "perp":
        return unipc or c["perp_refusal"] is not None
    if f == "fdg":
        # (the size rule, more than 5 levels, and a [B', N] tensor for a batch of B)
        return c["fdg_levels"] > fdg_max_levels(c["shape"]) or c["fdg_form"] == "bad_rows"
    if f in ("cfgzero", "tcfg"):
        if unipc:
            return c["guidance"] == "per_sample" and c["B"] > 1
        return f == "cfgzero" and c["method"] == "adaptive" and c["zero_init"] > 0
    if f == "cfgpp":
        return (unipc or c["algo"] != "dpmsolver++" or c["method"] != "multistep" or c["order"] not in (1, 2)
                or c["thresholding"])
    return unipc


# ---- the reference ---------------------------------------------------------------------------------------------------

def _fp32(c):
    return c["state_dtype"] is None and c["model_dtype"] is None


def reference_expressible(c):
    """cfgzero, tcfg and fdg: fp32 DPM_Solver, not adaptive, a network the reference's wrappers take on its schedule;
    cfgpp: fp32, a network with a closed-form x0, no denoise_to_zero; mask: fp32 DPM_Solver on a VP schedule, not
    adaptive; perp: fp32 DPM_Solver on a VP schedule, not adaptive, the network's outputs row-major. Never inverse()."""
    if refused(c) or not _fp32(c) or c["inverse"] or c["sampler"] != "dpm" or c["method"] == "adaptive":
        return False
    sched, mt = c["schedule"], c["model_type"]
    if c["feature"] in ("cfgzero", "tcfg", "fdg"):
        return mt == sched if sched in ("flow", "edm") else mt in ("noise", "x_start", "v", "score")
    if c["feature"] == "cfgpp":
        return mt in ("noise", "x_start", "v", "score", "flow") and sched != "edm" and not c["denoise_to_zero"]
    if c["feature"] == "perp" and not row_major_outputs(c):
        return False
    return sched not in ("flow", "edm") and mt in ("noise", "x_start", "v", "score")


def row_major_outputs(c):
    """Whether the network's outputs are row-major: it returns row-major ones, or keeps a row-major x's layout."""
    x_cl = c["x_channels_last"] and really_channels_last(dict(c, channels_last=True))
    return not (c["net_layout"] == "cl" and really_channels_last(c)) and not (c["net_layout"] == "keep" and x_cl)


def _guided_net(c, rig):
    """A network for the reference's guidance_type="uncond" wrapper that returns the guided output of rig.net."""
    B = c["B"]
    uc, cond = torch.zeros(B, 1), torch.ones(B, 1)
    if c["feature"] == "fdg":
        import fdg_oracle
        return fdg_oracle.guided_net(rig.net, uc, cond, fdg_values(c))
    # (one scale as per-sample scales: a scale of 1 then gives out_c itself, as the product's bypass does, not
    # us + 1*(out_c - us))
    w = torch.tensor(c["scales"] or [c["cfg"]] * B, dtype=torch.float32)
    if c["feature"] == "tcfg":
        import tcfg_oracle
        return tcfg_oracle.guided_net(rig.net, uc, cond, w)
    from cfgzero_oracle import guided_net
    return guided_net(rig.net, uc, cond, w, c["zero_init"])


def _reference_uncond(c, rig, x):
    """The reference driving _guided_net(c, rig) through guidance_type="uncond" (cfgzero, tcfg, fdg)."""
    from gpu_configs import reference
    ref = reference()
    rns = reference_schedule(c)
    g = _guided_net(c, rig)
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


def _reference_perp(c, rig, x):
    """Perp-Neg in the reference: for a noise network perpneg_oracle.guided_net behind a guidance_type="uncond" wrapper,
    else test_perp_neg.reference_composed, both on rig's network, conditions and the drawn scales."""
    from perpneg_oracle import guided_net
    from test_perp_neg import reference_composed
    B, rns = c["B"], reference_schedule(c)
    uc, cond = torch.zeros(B, 1), perp_conditions(c, "cpu")
    n = [0]
    if c["model_type"] == "noise":
        from gpu_configs import reference
        ref, calls = reference(), []
        fn = ref.model_wrapper(guided_net(rig.net, uc, cond, c["scales"], calls), rns, model_type="noise")
    else:
        ref, _, composed = reference_composed(c["model_type"], c["K"], model=rig.net, batch=B, scales=c["scales"],
                                              rns=rns, condition=cond)
        calls = None

        def fn(xx, t):
            n[0] += 1
            return composed(xx, t)
    s = ref.DPM_Solver(fn, rns, algorithm_type=c["algo"],
                       correcting_x0_fn="dynamic_thresholding" if c["thresholding"] else None)
    s.thresholding_max_val, s.dynamic_thresholding_ratio = c["max_val"], c["ratio"]
    with contextlib.redirect_stdout(io.StringIO()):
        y = s.sample(x, **sample_kwargs(c))
    return y, len(calls) if calls is not None else n[0]


def _cfgpp_fp64(c, rig, x, rounded=False):
    """(y, evaluations): cfgpp_fp64 on the product's grid and fp32 marginals, the network's halves converted to x0 in
    fp64; `rounded`: an x_start output converted as the product converts it, in fp32 (see _reference_cfgpp)."""
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
    f32 = np.float32

    def x0(out, xx, i):
        if mt == "x_start" and rounded:
            # eps = (x - alpha*o)/sigma, then x0 = (x - sigma*eps)/alpha, each op rounded to fp32
            xf, a, s_ = xx.astype(f32), f32(al[i]), f32(sg[i])
            e = ((xf - a * out.astype(f32)) / s_).astype(f32)
            return ((xf - s_ * e) / a).astype(f32).astype(np.float64)
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


def _reference_cfgpp(c, rig, x):
    """(y, evaluations, tolerance): _cfgpp_fp64 and the relative distance the product may lie from it.

    That is CFGPP_TOL, plus for an x_start network the rounding of its conversion. The product takes an x_start output
    o to x0 as the reference's data prediction does: eps = (x - alpha*o)/sigma (:292), then x0 = (x - sigma*eps)/alpha
    (:439), each op in fp32. x - sigma*eps cancels down to alpha*o, so x0 carries an error of about u*|x|/alpha
    (u = 2^-24), where the transcription takes x0 = o exactly; the guided x0 carries (1 + 2|w|) times that, and the
    update after grid point i scales it by alpha_{i+1}. Where alpha_i is small -- a flow schedule starts at
    alpha_T = 1/N -- this amounts to 1e-4 of the result at a few steps, against 1e-6 for a velocity or noise network.
    The replay `rounded` measures it on the run itself: the same conversion rounded to fp32, the rest in fp64. The
    product rounds that conversion, and the state it reads, independently of the replay, so it may lie up to
    XSTART_ROUNDING times the replay's distance away (at most about twice, over the draws and grids tried)."""
    y, n = _cfgpp_fp64(c, rig, x)
    tol = CFGPP_TOL
    if c["model_type"] == "x_start":
        tol += XSTART_ROUNDING * rel_err(_cfgpp_fp64(c, rig, x, rounded=True)[0], y)
    return y, n, tol


def reference_run(c, rig):
    """(y, number of evaluations, tolerance) of the reference form of `c` on rig's network; the tolerance is None where
    the product must match it bit for bit."""
    x = rig.x()
    if c["feature"] == "cfgpp":
        return _reference_cfgpp(c, rig, x)
    run = {"cfgzero": _reference_uncond, "tcfg": _reference_uncond, "fdg": _reference_uncond,
           "mask": _reference_mask, "perp": _reference_perp}[c["feature"]]
    return run(c, rig, x) + (None,)


def cpu_oracle(c):
    """{"y", "inter", "calls"} of the exact executor, plus "pinned" (the distance to the reference) when it was
    compared; {"error": exception} when the product refuses the configuration."""
    import dpm_solver_b200 as new
    out = {}
    with backend(executor(c)) as be:
        rig = None
        try:
            rig = GuidanceRig(new, c)
            out["y"], out["inter"], out["calls"] = rig.sample(rig.solver(), rig.x(), trace=True)
        except (ValueError, AssertionError) as e:
            # a refusal comes before any launch and any network call
            assert be.launch_count() == 0 and not getattr(rig, "trace_log", None), (c, e)
            return {"error": e}
        if c["fdg_equal"]:
            # equal scales: the pyramid terms vanish, so the run is the one-level run's bit for bit
            one = GuidanceRig(new, dict(c, fdg_levels=1, fdg_w=[r[:1] for r in c["fdg_w"]]))
            assert same_bits(out["y"], one.sample(one.solver(), one.x())[0]), c
        if reference_expressible(c):
            yr, n, tol = reference_run(c, GuidanceRig(new, c))
            assert len(out["calls"]) == n, (c, len(out["calls"]), n)
            if tol is not None:
                out["pinned"] = rel_err(out["y"], yr)
                assert out["pinned"] <= tol, (c, out["pinned"], tol)
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
    if f in ("tcfg", "fdg", "perp"):
        keys += [f + ":" + k for k in keys if k.startswith("layout change:")]
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
    elif f == "tcfg":
        bypass = c["guidance"] != "per_sample" and c["cfg"] == 1.0 or c["scales"] == [1.0]
        if bypass:
            keys.append("tcfg:bypass")
        elif c["sampler"] == "unipc" or (c["thresholding"] and c["algo"] == "dpmsolver++"):
            keys.append("tcfg:materialised")
        if c["guidance"] == "per_sample" and c["B"] > 1 and 1.0 in c["scales"]:
            keys.append("tcfg:per-sample row at 1")
    elif f == "fdg":
        H, W = c["shape"][-2:]
        # (g follows the network's outputs: channels_last ones, asked for or kept from a channels_last x, are strided
        # planes)
        strided = (x_cl and c["net_layout"] == "keep") or (c["net_layout"] == "cl" and really_channels_last(c))
        keys += ["fdg:levels=%d" % c["fdg_levels"],
                 "fdg:scales:" + {"bf16": "converted", "cpu": "converted"}.get(c["fdg_form"], c["fdg_form"])]
        if (H * W) % 8 or strided:
            keys.append("fdg:scalar path")
        if ps // (H * W) > 1:
            keys.append("fdg:planes>1 per sample")
        if c["fdg_equal"] and c["fdg_levels"] > 1:
            keys.append("fdg:equal scales")
    elif f == "perp":
        keys.append("perp:K=%d" % c["K"])
        if ps % 8:
            keys.append("perp:words element path")
        if ps > 8192:
            keys.append("perp:words multi-chunk")
        if c["perp_d1_zero"] is not None:
            keys.append("perp:|d1|=0")
        keys += ["perp:" + k for k in ("inverse", "d2z") if k in keys]
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
            ["inverse", "d2z", "t_start/t_end"] +
            ["tcfg:bypass", "tcfg:per-sample row at 1", "tcfg:materialised"] +
            ["fdg:levels=1", "fdg:levels=5", "fdg:scalar path", "fdg:planes>1 per sample", "fdg:equal scales"] +
            ["fdg:scales:" + k for k in ("floats", "listed", "vec", "rows", "converted")] +
            ["perp:K=%d" % k for k in (2, 3, 4)] +
            ["perp:" + k for k in ("words element path", "words multi-chunk", "|d1|=0", "inverse", "d2z")] +
            [f + ":layout change:" + k for f in ("tcfg", "fdg", "perp")
             for k in ("row-major outputs of a channels_last state", "channels_last outputs of a row-major state")])
REQUIRED_ON_DEVICE = ["rejected", "captured", "captured:zero-init", "captured:rewritten-mask", "second_stream",
                      "pinned", "fdg:frozen step served", "fdg:frozen step fell back", "captured:fdg rows rewritten"]


def configurations(chunk):
    rng = random.Random(SEED + chunk)
    return [draw_guidance(rng) for _ in range(PER_CHUNK)]
