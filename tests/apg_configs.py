"""Random adaptive-projected-guidance `sample()` configurations for the end-to-end tests on the device
(tests/test_gpu_apg_random_configs.py) and their CPU side (tests/test_apg_draws_vs_reference.py): the draw
(flow_unipc_configs.draw_flow_unipc, extended), an `APGRig` and the CPU oracle.

The draw adds an EDM schedule, apg_eta in {0, 0.3, 1}, a norm threshold that is off, always clips or never clips,
apg_momentum in {0, -0.5, 0.3}, one scale or per-sample scales with rows at 1, shapes of more than 8192 elements per
sample and of sizes that are not multiples of 8, a channels_last x_T, networks that return channels_last or row-major
outputs whatever their input (so that the state and the network outputs are in different layouts), and inverse().

The oracle of a configuration, on CPU tensors:
  * the product's host logic on the numpy executor with exact words (`APGOracle(exact=True)`): y, every intermediate and
    the trace of network calls -- what the device must give bit for bit;
  * where the unmodified reference can express the configuration (fp32, one scale, DPM_Solver not adaptive, or UniPC
    bh2 of order <= 2 without the corrector, which is its multistep DPM-Solver(++)(2M)), the executor must lie within
    REF_TOL of `apg_oracle.reference_solver` (the reference driven by an fp64 APG data prediction) with as many network
    calls;
  * a configuration the product refuses is {"error": exception}.
"""
import contextlib
import io
import random

import torch

from apg_oracle import APGOracle, apg_x0_model, reference_solver
from cases import make_betas
from flow_unipc_configs import FlowRig, draw_flow_unipc
from flow_unipc_configs import refused as flow_unipc_refused
from gpu_configs import DT, backend, really_channels_last, reference, rel_err, sample_kwargs

REF_TOL = 1e-4          # tests/test_apg.py: the reference reads an x0 formed in fp64, the product forms it op by op
PARAM = {"noise": 0, "x_start": 1, "v": 2, "score": 3, "flow": 4, "edm": 5}
# 16384 per sample (two chunks, whole packets, the pipeline quantile), 8235 (two chunks, not a multiple of 8), 8256
# (two chunks, whole packets), 105 and 35 (element-wise words, scalar step), 240 (whole packets, one chunk)
SHAPES = [(4, 64, 64), (3, 45, 61), (4, 48, 43), (3, 5, 7), (1, 7, 5), (3, 8, 10)]
THRESHOLDS = {"off": 0.0, "clips": 1e-3, "never": 1e6}
CHUNKS, PER_CHUNK, SEED = 6, 20, 9700     # the device test: 6 chunks of 20 configurations


def draw_apg(rng):
    c = draw_flow_unipc(rng)
    if rng.random() < 0.2:
        c.update(schedule="edm", model_type="edm", sigma_data=rng.choice([0.5, 1.0]))
    if not c["thresholding"]:
        c["shape"] = rng.choice(SHAPES)
        c["B"] = rng.choice([1, 2, 3, 4])
    c["apg_eta"] = rng.choice([0.0, 0.3, 1.0])
    c["apg_thr"] = rng.choice(list(THRESHOLDS))
    c["apg_momentum"] = rng.choice([0.0, -0.5, 0.3])
    g = rng.random()
    if g < 0.5:
        c.update(guidance="float", cfg=rng.choice([1.0, 3.5, 7.5, 7.5]), scales=None)
    elif g < 0.8:
        c.update(guidance="per_sample", cfg=None, scales=[rng.choice([7.5, 1.0, 3.5, -2.0]) for _ in range(c["B"])])
    elif g < 0.9:
        c.update(guidance="tensor0", cfg=rng.choice([3.5, 7.5]), scales=None)
    # (else draw_gpu's: none, multi or rescale now and then -- APG refuses them)
    if c["sampler"] == "unipc" and c["guidance"] == "per_sample" and rng.random() < 0.7:
        c.update(guidance="float", cfg=7.5, scales=None)       # (UniPC refuses per-sample scales)
    c["x_channels_last"] = len(c["shape"]) == 3 and rng.random() < 0.25
    c["net_layout"] = rng.choice(["keep", "keep", "cl", "row"]) if len(c["shape"]) == 3 else "keep"
    c["channels_last"] = c["net_layout"] == "cl"
    c["inverse"] = (c["sampler"] == "unipc" or c["method"] != "adaptive") and rng.random() < 0.15
    if c["inverse"]:
        c.update(t_start=None, t_end=None)
    return c


class APGRig(FlowRig):
    """FlowRig with an EDM schedule, APG in model_wrapper, a channels_last x_T and a network whose output layout is
    fixed (channels_last or row-major) or follows its input."""

    def __init__(self, mod, c, device="cpu"):
        self.mod, self.c, self.device, self.calls = mod, c, torch.device(device), None
        self.ns = self.make_schedule()
        B, md, lay = c["B"], DT[c["model_dtype"]], c["net_layout"]

        def net(xx, tt, cc=None):
            if self.calls is not None:
                self.calls.append((float(tt[0]), tuple(xx.shape)))
            one = (-1,) + (1,) * (xx.dim() - 1)
            o = 0.1 * xx.float() + ((tt * 0.001) * 0.05 - 0.02).reshape(one)      # cases.exact_net, any rank
            if cc is not None:
                o = o * (1. + 0.25 * cc.reshape(one)) + 0.05 * cc.reshape(one)
            if md is not None:
                o = o.to(md)
            if lay == "cl" and o.dim() == 4:
                return o.contiguous(memory_format=torch.channels_last)
            return o.contiguous() if lay == "row" else o

        self.net = net
        g = c["guidance"]
        apg = dict(apg_eta=c["apg_eta"], apg_norm_threshold=THRESHOLDS[c["apg_thr"]], apg_momentum=c["apg_momentum"])
        if g == "none":
            self.fn = mod.model_wrapper(lambda xx, tt: net(xx, tt), self.ns, model_type=c["model_type"], **apg)
            return
        kw = dict(model_type=c["model_type"], guidance_type="classifier-free",
                  unconditional_condition=torch.zeros(B, 1, device=self.device), **apg)
        if c["phi"]:
            kw["guidance_rescale"] = c["phi"]
        if g == "multi":
            cond = [torch.full((B, 1), float(k + 1), device=self.device) for k in range(len(c["scales"]))]
            scale = list(c["scales"])
        else:
            cond = torch.ones(B, 1, device=self.device)
            scale = c["cfg"]
            if g == "tensor0":
                scale = torch.tensor(c["cfg"])
            elif g == "per_sample":
                scale = torch.tensor(c["scales"], dtype=torch.float32, device=self.device)
        self.scale = scale
        self.fn = mod.model_wrapper(net, self.ns, condition=cond, guidance_scale=scale, **kw)

    def make_schedule(self):
        if self.c["schedule"] == "edm":
            return self.mod.NoiseScheduleEDM(sigma_data=self.c["sigma_data"])
        return super().make_schedule()

    def x(self):
        x = super().x()
        return x.contiguous(memory_format=torch.channels_last) if self.c["x_channels_last"] else x

    def sample(self, s, x, trace=False, **over):
        if not self.c["inverse"]:
            return super().sample(s, x, trace, **over)
        kw = dict(self.kwargs(), **over)
        kw = {k: v for k, v in kw.items() if k not in ("use_corrector", "atol", "rtol")}
        self.calls = [] if trace else None
        try:
            y, inter = s.inverse(x, return_intermediate=True, **kw)
            return y, inter, self.calls
        finally:
            self.calls = None


def refused(c):
    """Whether the product must refuse `c` with a ValueError before any launch."""
    if flow_unipc_refused(c) or c["guidance"] in ("none", "multi") or c["phi"]:
        return True
    if c["schedule"] == "edm" and c["reference_rounding"]:
        return True
    return c["sampler"] == "dpm" and c["method"] == "adaptive" and c["apg_momentum"] != 0


# ---- the reference ---------------------------------------------------------------------------------------------------

def reference_expressible(c):
    """fp32, one scale (a per-sample vector at B = 1 is one scale), DPM_Solver not adaptive or UniPC bh2-2M."""
    if c["state_dtype"] is not None or c["model_dtype"] is not None or c["inverse"]:
        return False
    if c["guidance"] == "per_sample" and c["B"] > 1:
        return False
    if c["sampler"] == "unipc":
        return (c["variant"] == "bh2" and c["order"] <= 2 and not c["use_corrector"] and c["steps"] >= c["order"]
                and not (c["order"] == 2 and c["lower_order_final"] and c["steps"] >= 10))
    return c["method"] != "adaptive"


def reference_schedule(c):
    ref = reference()
    if c["schedule"] == "edm":
        from edm_oracle import reference_schedule as edm
        return edm(sigma_data=c["sigma_data"])
    if c["schedule"] == "flow":
        from flow_oracle import reference_schedule as flow
        return flow(c["shift"], c["time_scale"])
    kind, betas = make_betas(c["schedule"])
    return ref.NoiseScheduleVP("linear") if kind == "linear" else \
        ref.NoiseScheduleVP("discrete", betas=torch.from_numpy(betas))


def reference_run(c, rig):
    """(y, number of network calls) of the unmodified reference on `c`, its data prediction APG in fp64 through
    `rig.net` (a UniPC configuration runs as multistep DPM-Solver)."""
    if c["sampler"] == "unipc":
        c = dict(c, method="multistep", solver_type="dpmsolver")
    rns = reference_schedule(c)
    tin = getattr(rns, "input_time", None)
    if tin is None:
        tin = (lambda t: (t - 1. / rns.total_N) * 1000.) if getattr(rns, "schedule", "") == "discrete" else (lambda t: t)
    B = c["B"]
    w = c["cfg"] if c["guidance"] != "per_sample" else c["scales"][0]
    x0_fn = apg_x0_model(rig.net, rns, PARAM[c["model_type"]], torch.zeros(B, 1), torch.ones(B, 1), float(w),
                         c["apg_eta"], THRESHOLDS[c["apg_thr"]], c["apg_momentum"], tin)
    s = reference_solver(rns, x0_fn, c["algo"], c["thresholding"])
    s.thresholding_max_val, s.dynamic_thresholding_ratio = c["max_val"], c["ratio"]
    rig.calls = []
    with contextlib.redirect_stdout(io.StringIO()):
        y = s.sample(rig.x(), **sample_kwargs(c))
    return y, len(rig.calls)


def cpu_oracle(c):
    """{"y", "inter", "calls"} of the exact executor, plus "pinned": the reference's relative distance when it was
    compared; {"error": exception} when the product refuses the configuration."""
    import dpm_solver_b200 as new
    out = {}
    with backend(APGOracle(exact=True)):
        try:
            rig = APGRig(new, c)
            out["y"], out["inter"], out["calls"] = rig.sample(rig.solver(), rig.x(), trace=True)
        except (ValueError, AssertionError) as e:
            return {"error": e}
    if reference_expressible(c):
        yr, ncalls = reference_run(c, APGRig(new, c))
        assert len(out["calls"]) == ncalls, c
        out["pinned"] = rel_err(out["y"], yr)
        assert out["pinned"] <= REF_TOL, (c, out["pinned"])
    return out


# ---- the tally -------------------------------------------------------------------------------------------------------

def per_sample(c):
    n = 1
    for d in c["shape"]:
        n *= d
    return n


def tally_static(c):
    """Entries that follow from a configuration the product accepts (also computed without a device)."""
    ps = per_sample(c)
    keys = ["schedule:" + ("vp" if c["schedule"] not in ("flow", "edm") else c["schedule"]), "sampler:" + c["sampler"],
            "eta:%g" % c["apg_eta"], "threshold:" + c["apg_thr"], "momentum:%g" % c["apg_momentum"]]
    if ps > 8192:
        keys.append("words:multi-chunk")
    if ps % 8:
        keys += ["words:element-wise", "step:scalar"]
    if c["thresholding"]:
        keys.append("quantile:pipeline" if ps >= 8192 else "quantile:cluster")
    if c["guidance"] == "per_sample" and c["B"] > 1 and 1.0 in c["scales"]:
        keys.append("bypassed row")
    if c["state_dtype"]:
        keys.append("state:16-bit")
    if c["x_channels_last"] and really_channels_last(dict(c, channels_last=True)):
        keys.append("x:channels_last")
        if c["net_layout"] == "row":
            keys.append("layout change:row-major outputs of a channels_last state")
    if c["net_layout"] == "cl" and not c["x_channels_last"] and really_channels_last(c):
        keys.append("layout change:channels_last outputs of a row-major state")
    if any(k.startswith("layout change") for k in keys) and c["apg_momentum"]:
        keys.append("momentum across a layout change")
    if c["sampler"] == "dpm":
        keys.append("method:" + c["method"])
    if c["inverse"]:
        keys.append("inverse")
    if c["denoise_to_zero"]:
        keys.append("d2z")
    if c["t_start"] is not None or c["t_end"] is not None:
        keys.append("t_start/t_end")
    return keys


REQUIRED = (["schedule:" + s for s in ("vp", "flow", "edm")] + ["sampler:dpm", "sampler:unipc"] +
            ["eta:0", "eta:0.3", "eta:1", "threshold:off", "threshold:clips", "threshold:never", "momentum:0",
             "momentum:-0.5", "momentum:0.3", "words:multi-chunk", "words:element-wise", "step:scalar",
             "quantile:pipeline", "quantile:cluster", "bypassed row", "state:16-bit", "x:channels_last",
             "layout change:row-major outputs of a channels_last state",
             "layout change:channels_last outputs of a row-major state", "momentum across a layout change",
             "method:singlestep", "method:singlestep_fixed",
             "method:adaptive", "method:multistep", "inverse", "d2z", "t_start/t_end"])
REQUIRED_ON_DEVICE = ["rejected", "captured", "captured:momentum", "second_stream", "pinned"]


def configurations(chunk):
    rng = random.Random(SEED + chunk)
    return [draw_apg(rng) for _ in range(PER_CHUNK)]
