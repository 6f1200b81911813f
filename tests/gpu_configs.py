"""Random `sample()` configurations for the end-to-end tests on the device (tests/test_gpu_random_configs.py,
tests/test_gpu_solver_reuse.py): the draw (`draw_wide` of test_random_configs_vs_reference.py, extended), one `Rig` per
(module, configuration, device) that builds the schedule, the network, `model_fn` and solvers, and the two CPU oracles.

The oracles of a configuration, both on CPU tensors:
  * the unmodified reference (oracle/_ref), whenever it can express the configuration: fp32 state and network, one
    guidance scale or none;
  * the product's host logic on the numpy executor (`FullOracle`), for everything: 16-bit state, per-sample scales,
    guidance rescale, several conditions (each pinned to the reference by the CPU tests of its feature).
The network is made of exact IEEE multiplies and adds (cases.exact_net written for any rank, plus condition terms), so a
CPU and a CUDA evaluation return the same bits."""
import contextlib
import io
import random

import numpy as np
import torch

from cases import make_betas, seeded
from oracle import ref_loader
from test_cfg_multi import MultiOracle
from test_cfg_per_sample import GuidedOracle
from test_random_configs_vs_reference import draw_wide

DT = {None: None, "bf16": torch.bfloat16, "f16": torch.float16}
# tiny shapes (scalar kernel, cluster quantile); [B,4,64,64] (packet kernels, whole 32 KB tiles of the duplicating
# kernels, pipeline quantile at 16384 per sample); 4800 per sample (not a multiple of the 4096-element tile); 105 per
# sample (neither it nor B*105 is a multiple of 8, B in 1, 2, 3, 5); one 5-D shape
SHAPES = [(1, 7, 5), (3, 8, 8), (4, 64, 64), (4, 64, 64), (3, 40, 40), (3, 5, 7), (2, 3, 6, 4)]
GUIDANCE = ["none", "none", "float", "float", "tensor0", "per_sample", "multi", "rescale"]
PHI = 0.7
CHUNKS, PER_CHUNK, SEED = 8, 25, 9000     # the device test: 8 chunks of 25 configurations


class FullOracle(GuidedOracle, MultiOracle):
    """The numpy executor with every guidance form: per-sample scales and the rescale (GuidedOracle), several
    conditions and `replicate` (MultiOracle)."""


@contextlib.contextmanager
def backend(be):
    from dpm_solver_b200 import ops
    old = ops._backend
    ops.set_backend(be)
    try:
        yield be
    finally:
        ops.set_backend(old)


def draw_gpu(rng):
    """draw_wide() plus the shapes above, a channels_last network, 16-bit state / network, every guidance form and the
    kernel variant."""
    c = draw_wide(rng)
    c["shape"] = rng.choice(SHAPES)
    c["B"] = rng.choice([1, 4]) if c["shape"] == (4, 64, 64) else rng.choice([1, 2, 3, 5])
    c["channels_last"] = len(c["shape"]) == 3 and rng.random() < 0.2
    c["x2_channels_last"] = len(c["shape"]) == 3 and not c["channels_last"] and rng.random() < 0.15
    c["state_dtype"] = rng.choice([None, None, "bf16", "f16"])
    c["model_dtype"] = c["state_dtype"] or rng.choice([None, None, None, "bf16"])
    kind = c["guidance"] = rng.choice(GUIDANCE)
    c["cfg"] = None if kind in ("none", "per_sample", "multi") else rng.choice([1.0, 3.5, 7.5, 7.5])
    c["scales"] = None
    if kind == "per_sample":
        c["scales"] = [rng.choice([7.5, 1.0, 0.0, -2.0, 3.5]) for _ in range(c["B"])]
    elif kind == "multi":
        c["scales"] = [rng.choice([4.0, 0.0, -1.5, 7.5]) for _ in range(rng.choice([2, 3]))]
    # (the rescale with several conditions is a combination model_wrapper rejects)
    c["phi"] = PHI if kind == "rescale" or (kind in ("per_sample", "multi") and rng.random() < 0.15) else 0.0
    c["tuning"] = rng.choice(["auto", "auto", "tma"])
    return c


def reference_expressible(c):
    """True when the unmodified reference computes this configuration (fp32 throughout, at most one scale)."""
    return (c["state_dtype"] is None and c["model_dtype"] is None and c["guidance"] in ("none", "float", "tensor0")
            and c["phi"] == 0.0)


def really_channels_last(c):
    """Whether channels_last is another memory order than row-major for this shape (not with one channel or 1x1)."""
    t = torch.empty((c["B"],) + tuple(c["shape"]))
    return c["channels_last"] and not t.contiguous(memory_format=torch.channels_last).is_contiguous()


def freezable(c):
    """Whether some step of the configuration is one `ops.PreparedStep.build` accepts: a fixed-grid method, every
    operand row-major, and no per-sample data (thresholds, rescale ratios, per-sample scales) or several conditions."""
    guided = c["guidance"] in ("per_sample", "multi") or (c["guidance"] == "rescale" and c["cfg"] != 1.0)
    return c["method"] != "adaptive" and not c["thresholding"] and not guided and not really_channels_last(c)


def sample_kwargs(c):
    kw = dict(steps=c["steps"], order=c["order"], skip_type=c["skip_type"], method=c["method"],
              lower_order_final=c["lower_order_final"], denoise_to_zero=c["denoise_to_zero"], solver_type=c["solver_type"],
              t_end=c["t_end"], t_start=c["t_start"])
    if c["method"] == "adaptive":
        kw.update(atol=c["atol"], rtol=c["rtol"])
    return kw


class Rig:
    """Schedule, network, model_fn and solvers of configuration `c` in module `mod` (the product or the reference) on
    `device`. `calls`, when a list, receives (first time label, input shape) of every network call; None records
    nothing and reads nothing back (graph capture, sync-free runs)."""

    def __init__(self, mod, c, device="cpu"):
        self.mod, self.c, self.device, self.calls = mod, c, torch.device(device), None
        self.ns = self.make_schedule()
        B, md, cl = c["B"], DT[c["model_dtype"]], c["channels_last"]

        def net(xx, tt, cc=None):
            if self.calls is not None:
                self.calls.append((float(tt[0]), tuple(xx.shape)))
            one = (-1,) + (1,) * (xx.dim() - 1)
            o = 0.1 * xx.float() + ((tt * 0.001) * 0.05 - 0.02).reshape(one)      # cases.exact_net, any rank
            if cc is not None:
                o = o * (1. + 0.25 * cc.reshape(one)) + 0.05 * cc.reshape(one)    # (so that std(out_c) != std(out_u))
            if md is not None:
                o = o.to(md)
            return o.contiguous(memory_format=torch.channels_last) if cl else o

        self.net = net
        g = c["guidance"]
        if g == "none":
            self.fn = mod.model_wrapper(lambda xx, tt: net(xx, tt), self.ns, model_type=c["model_type"])
            return
        kw = dict(model_type=c["model_type"], guidance_type="classifier-free",
                  unconditional_condition=torch.zeros(B, 1, device=self.device))
        if c["phi"]:
            kw["guidance_rescale"] = c["phi"]
        if g == "multi":
            cond = [torch.full((B, 1), float(k + 1), device=self.device) for k in range(len(c["scales"]))]
            scale = list(c["scales"])
        else:
            cond = torch.ones(B, 1, device=self.device)
            scale = c["cfg"]
            if g == "tensor0" and mod.__name__ == "dpm_solver_b200":
                scale = torch.tensor(c["cfg"])              # (the reference takes the python float)
            elif g == "per_sample":
                scale = torch.tensor(c["scales"], dtype=torch.float32, device=self.device)
        self.scale = scale
        self.fn = mod.model_wrapper(net, self.ns, condition=cond, guidance_scale=scale, **kw)

    @property
    def calls(self):
        return self.__dict__.get("_calls")

    @calls.setter
    def calls(self, v):
        """A list set here is also kept as `trace_log` after sample() lets go of it, so that a call that raised can be
        checked for network calls."""
        self._calls = v
        if v is not None:
            self.trace_log = v

    def make_schedule(self):
        kind, betas = make_betas(self.c["schedule"])
        return self.mod.NoiseScheduleVP("linear") if kind == "linear" else \
            self.mod.NoiseScheduleVP("discrete", betas=torch.from_numpy(betas))

    def solver(self, **kw):
        c = self.c
        if self.mod.__name__ == "dpm_solver_b200":
            kw.setdefault("state_dtype", DT[c["state_dtype"]])
        return self.mod.DPM_Solver(self.fn, self.ns, algorithm_type=c["algo"],
                                   correcting_x0_fn="dynamic_thresholding" if c["thresholding"] else None,
                                   thresholding_max_val=c["max_val"], dynamic_thresholding_ratio=c["ratio"], **kw)

    def x(self):
        c = self.c
        return (seeded((c["B"],) + tuple(c["shape"]), c["seed"]) * c["scale"]).to(self.device)

    def x2(self):
        """A second input of the same shape: 0.5 * x + other values (channels_last when the configuration says so)."""
        c = self.c
        x2 = 0.5 * self.x() + seeded((c["B"],) + tuple(c["shape"]), c["seed"] + 1).to(self.device)
        return x2.contiguous(memory_format=torch.channels_last) if c["x2_channels_last"] else x2

    def sample(self, s, x, trace=False, **over):
        """(y, intermediates, calls) of `s.sample(x)`; the adaptive method has no intermediates (and prints)."""
        kw = dict(sample_kwargs(self.c), **over)
        self.calls = [] if trace else None
        try:
            if kw["method"] == "adaptive":
                with contextlib.redirect_stdout(io.StringIO()):
                    y, inter = s.sample(x, **kw), []
            else:
                y, inter = s.sample(x, return_intermediate=True, **kw)
            return y, inter, self.calls
        finally:
            self.calls = None


def same_bits(a, b):
    """Same dtype, shape and bit patterns; NaNs must sit in the same places (their payloads are not compared)."""
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    nan = a.isnan()
    if not torch.equal(nan, b.isnan()):
        return False
    bits = torch.int32 if a.dtype == torch.float32 else torch.int16
    z = torch.zeros((), dtype=a.dtype)
    return torch.equal(torch.where(nan, z, a).view(bits), torch.where(nan, z, b).view(bits))


def rel_err(a, b):
    a, b = a.detach().double().cpu().numpy(), b.detach().double().cpu().numpy()
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def reference():
    import warnings
    warnings.filterwarnings("ignore")
    return ref_loader.load("dpm_solver_pytorch")


def cpu_oracle(c):
    """The CPU result the device must reproduce: {"y", "inter", "calls"} of the numpy executor, checked bit for bit
    (trace of network calls included) against the unmodified reference wherever the reference can express `c`;
    {"error": exception} when the configuration is rejected (by both, with the same exception type)."""
    import dpm_solver_b200 as new
    out = {}
    with backend(FullOracle()):
        try:
            rig = Rig(new, c)
            out["y"], out["inter"], out["calls"] = rig.sample(rig.solver(), rig.x(), trace=True)
        except (ValueError, AssertionError) as e:      # a rejected configuration: the device run must refuse it too
            out = {"error": e}
    if not reference_expressible(c):
        return out
    try:
        rig = Rig(reference(), c)
        yr, ir, cr = rig.sample(rig.solver(), rig.x(), trace=True)
    except Exception as e:
        assert "error" in out and type(out["error"]) is type(e), (c, e, out.get("error"))
        return out
    assert "error" not in out, (c, out.get("error"))
    if c["method"] == "adaptive":       # (its error norm sums in another order: tests/test_adaptive.py)
        assert len(out["calls"]) == len(cr), c
        return out
    assert out["calls"] == cr, c
    assert same_bits(out["y"], yr) and len(out["inter"]) == len(ir), c
    assert all(same_bits(a, b) for a, b in zip(out["inter"], ir)), c
    out["reference"] = True
    return out


def tally_static(c):
    """Entries that follow from the configuration alone (also computed without a device, to tune the draw)."""
    keys = ["guidance:" + c["guidance"], "state:" + str(c["state_dtype"]), "model:" + str(c["model_dtype"])]
    cfg = c["guidance"] in ("per_sample", "multi") or (c["cfg"] is not None and c["cfg"] != 1.0)
    if c["thresholding"]:
        n = 1
        for d in c["shape"]:
            n *= d
        keys.append("quantile:pipeline" if n >= 8192 else "quantile:cluster")
    if c["denoise_to_zero"]:
        keys.append("d2z:cfg" if cfg else "d2z:plain")
    if c["method"] == "multistep" and c["steps"] < 10 and c["lower_order_final"]:
        keys.append("multistep%d:lower_order_final" % c["order"])
    if c["method"] == "singlestep" and c["order"] == 3:
        keys.append("singlestep3:steps%%3=%d" % (c["steps"] % 3))
    if c["tuning"] == "tma":
        keys.append("tuning:tma")
    if really_channels_last(c):
        keys.append("channels_last")
    if c["x2_channels_last"]:
        keys.append("x2:channels_last")
    keys.append("method:" + c["method"])
    return keys


REQUIRED = (["guidance:" + g for g in ("none", "float", "tensor0", "per_sample", "multi", "rescale")] +
            ["state:None", "state:bf16", "state:f16", "model:bf16", "quantile:pipeline", "quantile:cluster", "d2z:cfg",
             "d2z:plain", "multistep1:lower_order_final", "multistep2:lower_order_final", "multistep3:lower_order_final",
             "singlestep3:steps%3=0", "singlestep3:steps%3=1", "singlestep3:steps%3=2", "tuning:tma", "channels_last",
             "method:adaptive", "method:singlestep_fixed"])
REQUIRED_ON_DEVICE = ["prepared:dup", "prepared:plain", "prepared:fell_back", "captured", "rejected", "second_stream"]


def configurations(chunk):
    """The configurations of one chunk of the device test."""
    rng = random.Random(SEED + chunk)
    return [draw_gpu(rng) for _ in range(PER_CHUNK)]
