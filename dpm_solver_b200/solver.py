"""Drop-in `model_wrapper` and `DPM_Solver` (reference: dpm_solver_pytorch.py:170-334, :337-1245).

Same names, positional order, defaults, return types and error behaviour as the reference; the
per-step arithmetic runs as fused sm_90a kernels behind the C-ABI (ops.py). What changes under
the hood:

* all schedule scalars come from the host-side plan (plan.py) -- no per-step interpolation
  kernels and no `.item()` syncs inside the loop;
* the conversion of the raw network output (x_start/v/score parameterisation :288-298, CFG
  combine :329-330, eps->x0 :439, thresholding clamp :424) is fused with the solver update that
  consumes it: one kernel per model evaluation reads (x, eps[, eps_uncond], older buffers) and
  writes (buffered model value, x_next);
* dynamic thresholding's per-sample quantile (:422) is one exact radix-select launch.

The order of model evaluations, their (x, t) arguments, the hooks (`correcting_x0_fn`,
`correcting_xt_fn`) and `return_intermediate` are those of the reference.
"""
from __future__ import annotations

import contextlib
import dataclasses
import inspect
import math
from dataclasses import dataclass
from typing import List, NamedTuple, Optional

import torch
import torch.distributed as dist

from . import ops, plan as P
from ._lib import FORM_LIN1, FORM_NONE, FORM_SS3T, PARAM_BY_NAME, PARAM_EDM, PARAM_FLOW, PARAM_NOISE
from .ops import StepArgs

__all__ = ["model_wrapper", "DPM_Solver", "WrappedModel"]

_DEV = object()     # marker: the scalars of this evaluation live in device memory (on-device adaptive controller)


# =================================================================================================
# model_wrapper
# =================================================================================================

class _Option(NamedTuple):
    name: str           # as messages name it
    combine: bool       # a guidance form of the combine: it runs with no other form but those _JOINED with it
    per_sample: bool    # takes per-sample guidance scales
    needs_uc: bool      # needs guidance_type='classifier-free' and an unconditional_condition
    refuses: str        # the solver contexts (_CONTEXTS) it does not run in


# The guidance options and what each runs with. A refused pair names the later option first, so this order decides
# which of several refusals a call reports. "sde" is DPM_Solver's algorithm_type, which refuses contexts as they do.
_OPTIONS = {
    "several": _Option("several conditions", True, False, False, "rr sde unipc"),
    "mask": _Option("guidance_mask", True, False, True, "rr sde unipc"),
    "perp": _Option("perp_neg", True, False, True, "rr sde unipc"),
    "rescale": _Option("guidance_rescale", True, True, False, "rr unipc"),
    "apg": _Option("adaptive projected guidance (apg_eta)", True, True, True, "rr sde"),
    "cfgzero": _Option("cfg_zero_star", True, True, True, "rr"),
    "cfgpp": _Option("cfg_pp", True, True, True, "rr sde unipc eps x0_fn adaptive singlestep order direct"),
    "tcfg": _Option("tcfg", True, True, True, "rr"),
    "fdg": _Option("fdg_scales", True, False, True, "rr"),
    "per_sample": _Option("a per-sample guidance_scale", False, True, False, "rr unipc"),
    "zero_init": _Option("cfg_zero_init_steps > 0", False, True, False, "adaptive"),
    "momentum": _Option("apg_momentum != 0", False, True, False, "adaptive"),
    "sde": _Option("algorithm_type='sde-dpmsolver++'", False, True, False, "rr adaptive singlestep direct inverse"),
}
_JOINED = ({"several", "mask"}, {"several", "perp"})     # the forms of the multi-condition combine
_CONTEXTS = {"rr": "reference_rounding=True", "sde": "algorithm_type='sde-dpmsolver++'", "unipc": "UniPC",
             "eps": "algorithm_type='dpmsolver'", "x0_fn": "dynamic thresholding or a correcting_x0_fn",
             "adaptive": "method='adaptive'", "inverse": "inverse()"}


def _check_options(options, contexts=(), what=None) -> None:
    """ValueError unless the guidance options `options` (keys of _OPTIONS) run together and in every solver context of
    `contexts`; `what` names the context in the message when _CONTEXTS does not."""
    active = [k for k in _OPTIONS if k in options]
    for i, k in enumerate(active):
        o = _OPTIONS[k]
        for j in active[:i]:
            p = _OPTIONS[j]
            if ((o.combine and p.combine and {j, k} not in _JOINED) or (k == "per_sample" and not p.per_sample)
                    or (j == "per_sample" and not o.per_sample)):
                raise ValueError("{} is not available with {}".format(o.name, p.name))
        for c in contexts:
            if c in o.refuses.split():
                raise ValueError("{} is not available with {}".format(o.name, what or _CONTEXTS[c]))


@dataclass
class RawOutput:
    """Network output(s) before parameterisation / guidance have been applied."""
    e_cond: torch.Tensor
    e_uncond: Optional[torch.Tensor]
    param: int
    guidance: float
    guidance_b: Optional[torch.Tensor] = None   # per-sample scales, fp32 [B] (then `guidance` is not read)
    # multi-condition guidance (K >= 2 conditions): the K conditional outputs in condition order (`e_cond` is the first)
    # and their fp32-rounded scales; `guidance` is then not read
    e_conds: Optional[tuple] = None
    scales: Optional[tuple] = None
    masks: Optional[tuple] = None   # regional guidance: one _CondMask or None (all ones) per condition, with e_conds
    is_x0: bool = False     # `e_cond` is a materialised x0 (a guided flow or EDM prediction): it is only clamped, not converted
    # the guidance form of the combine, a key of _OPTIONS ("" for plain guidance), and its host constants: (phi,) for
    # "rescale", (eta, norm_threshold, momentum) for "apg"
    form: str = ""
    consts: tuple = ()
    # frequency-decoupled guidance (form "fdg"): (scales, levels), the scales `levels` python floats or an fp32
    # [B, levels] tensor on the outputs' device; the solver turns the pair into one output g (dpm_fdg_guided)
    fdg: Optional[tuple] = None


def _multi_condition(condition, unconditional_condition, guidance_scale, masked=False):
    """model_wrapper's list or tuple of conditions -> (condition, guidance_scale, per-condition scales or None).
    One condition is the tensor form (its scale as one python float); K >= 2 conditions, or any K with guidance masks,
    keep their K scales, each read on the host once and rounded to fp32 once."""
    K = len(condition)
    if not 1 <= K <= ops._lib.MAX_CONDITIONS:
        raise ValueError("classifier-free guidance takes 1 to {} conditions, got {}".format(ops._lib.MAX_CONDITIONS, K))
    s = guidance_scale
    if not isinstance(s, (list, tuple)) and not (torch.is_tensor(s) and s.dim() >= 1):
        raise ValueError("a list of {} conditions needs a list, tuple or 1-D tensor of {} guidance scales, got a "
                         "single scale".format(K, K))
    s = torch.as_tensor(s.detach().cpu() if torch.is_tensor(s) else list(s), dtype=torch.float32)
    if s.dim() != 1:
        raise ValueError("a list of conditions takes one guidance scale per condition (shape [{}]); per-sample scales "
                         "are not available with several conditions, got shape {}".format(K, tuple(s.shape)))
    if s.numel() != K:
        raise ValueError("{} guidance scales for {} conditions".format(s.numel(), K))
    scales = tuple(s.tolist())
    if K == 1 and not masked:
        return condition[0], scales[0], None
    if unconditional_condition is None:
        raise ValueError("classifier-free guidance with {} conditions needs an unconditional_condition".format(K))
    return tuple(condition), scales, scales


class _CondMask:
    """One condition's guidance_mask. A mask that broadcasts to x's shape [B, C, *spatial] (batch extent 1 or B) becomes
    the weight map of dpm_step_multi_masked, once per (tensor, version, shape, storage order): period 1 when it is
    constant over every non-batch dim, a pixel map (period = spatial size) when it is constant over the channels of a
    row-major x, else an element map in x's storage order (channels_last included). Values are taken in fp32. A
    contiguous fp32 tensor on x's device that already has the map's layout is read in place, so a captured graph sees
    values written into it."""

    def __init__(self, mask: torch.Tensor):
        self.mask = mask
        self._cache = None

    def check(self, shape) -> None:
        """ValueError unless the mask broadcasts to `shape` (so its batch extent is 1 or shape[0])."""
        m = self.mask
        if m.dim() > len(shape) or any(a != 1 and a != b for a, b in zip(m.shape[::-1], tuple(shape)[::-1])):
            raise ValueError("guidance_mask of shape {} does not broadcast to x's shape {}".format(
                tuple(m.shape), tuple(shape)))

    def weights(self, shape, layout: str, device):
        """(w, period, sample_stride) for a launch over `shape` in storage order `layout` ('c' or 'cl') on `device`."""
        key = (id(self.mask), self.mask._version, tuple(shape), layout, str(device))
        if self._cache is None or self._cache[0] != key:
            self.check(shape)
            self._cache = (key, self._canonical(tuple(shape), layout, device))
        return self._cache[1]

    def _canonical(self, shape, layout, device):
        B, d = shape[0], len(shape)
        m = self.mask.detach()
        m = m.reshape((1,) * (d - m.dim()) + tuple(m.shape)).to(device=device, dtype=torch.float32)
        bm = m.shape[0]
        per_sample = math.prod(shape[1:])
        if all(v == 1 for v in m.shape[1:]):
            w, period = m.reshape(bm, 1), 1
        elif layout == "c" and d >= 3 and m.shape[1] == 1:
            period = math.prod(shape[2:])
            w = m.expand((bm, 1) + shape[2:]).reshape(bm, period)
        else:
            full = m.expand((bm,) + shape[1:])
            if layout == "cl":
                full = full.permute(0, *range(2, d), 1)      # channels_last storage order
            w, period = full.reshape(bm, per_sample), per_sample
        return w.contiguous(), period, (period if bm == B and B != 1 else 0)

    def rows(self, rows, x_dims: int) -> "_CondMask":
        """The mask of the batch rows `rows` of an x with `x_dims` dims (a mask shared by the batch is kept)."""
        m = self.mask
        if m.dim() < x_dims or m.shape[0] == 1:
            return self
        return _CondMask(m[rows])


def _words(be, raw: RawOutput) -> Optional[torch.Tensor]:
    """The per-sample words pass of a guided evaluation over both raw halves (2 launches; each sample's words read its
    own values only): the rescale ratio std(out_c)/std(g), CFG-Zero*'s s* or TCFG's (wu, wc). None for other forms."""
    if raw.form == "rescale":
        fn = getattr(be, "cfg_rescale_ratio", None)
        if fn is None:
            raise RuntimeError("guidance_rescale needs an executor with cfg_rescale_ratio; {} has none".format(
                getattr(be, "name", type(be).__name__)))
        return fn(raw.e_cond, raw.e_uncond, raw.guidance if raw.guidance_b is None else raw.guidance_b)
    if raw.form == "cfgzero":
        return be.cfgzero_scale(raw.e_cond, raw.e_uncond)
    if raw.form == "tcfg":
        return be.tcfg_words(raw.e_cond, raw.e_uncond)
    return None


def _guidance_args(a: StepArgs, words: Optional[torch.Tensor], raw: RawOutput, rows=None) -> StepArgs:
    """The guidance of `raw` on a step (rows `rows` of its per-sample fields): its per-sample words (`_words`), its
    per-sample scales, and the outputs, scales and masks of several conditions."""
    if words is not None:
        w = words if rows is None else words[rows]
        if raw.form == "rescale":
            a.ratio, a.phi = w, raw.consts[0]
        elif raw.form == "cfgzero":
            a.cfgzero_s = w
        else:
            a.tcfg_w = w
    if raw.guidance_b is not None and a.n_model == 2:
        a.guidance_b = raw.guidance_b if rows is None else raw.guidance_b[rows]
    if raw.e_conds is not None and a.n_model == 2:
        a.e_conds = raw.e_conds if rows is None else tuple(e[rows] for e in raw.e_conds)
        a.scales = raw.scales
        if raw.masks is not None:
            d = raw.e_cond.dim()
            a.masks = raw.masks if rows is None else tuple(m if m is None else _map_rows(m, rows, d) for m in raw.masks)
    if words is not None or a.guidance_b is not None or a.masks is not None:
        a.per_sample = a.e_cond.numel() // a.e_cond.shape[0]
    return a


def _map_rows(m, rows, x_dims: int):
    """The weight map of the batch rows `rows`: a _CondMask's own rows, or those of a (w, period, sample_stride) triple
    (a map shared by the batch, sample_stride 0, is kept)."""
    if isinstance(m, _CondMask):
        return m.rows(rows, x_dims)
    w, period, stride = m
    return m if stride == 0 else (w.reshape(-1, period)[rows].reshape(-1), period, stride)


def _perp_output(be, raw: RawOutput) -> RawOutput:
    """A Perp-Neg evaluation as an ordinary regional-guidance one: the words pass over the K+1 outputs (2 launches)
    gives condition 1's per-sample weight w_1, which becomes its period-1 weight map under the scales (1, s_2, ..., s_K);
    everything downstream is the masked multi-condition path."""
    fn = getattr(be, "perpneg_words", None)
    if fn is None:
        raise RuntimeError("perp_neg needs an executor with perpneg_words; {} has none".format(
            getattr(be, "name", type(be).__name__)))
    w = fn(raw.e_uncond, raw.e_conds, raw.scales)
    K = len(raw.scales)
    return dataclasses.replace(raw, scales=(1.0,) + tuple(raw.scales[1:]), masks=((w, 1, 1),) + (None,) * (K - 1),
                               form="")


def _apg_args(be, raw: RawOutput, xe, marg, sdtype, x0: bool, ns, coef_dev=None, r_prev=None, r_out=None) -> StepArgs:
    """StepArgs of an adaptive-projected-guidance evaluation of `raw`, its words computed (dpm_apg_words, 2 launches):
    both halves converted to x0 with the marginals `marg` = (alpha_t, sigma_t) (EDM: its x0 words), or with those of the
    device block `coef_dev` when `marg` is None; the guided x0 buffered when `x0`, else converted to eps with the same
    marginals. r_prev / r_out: the momentum buffer (read / written), or None."""
    eta, norm_threshold, momentum = raw.consts
    al, sg = marg if marg is not None else (1.0, 0.0)
    a = StepArgs(n_model=2, e_cond=raw.e_cond, e_uncond=raw.e_uncond, param=raw.param, guidance=raw.guidance,
                 predict_x0=x0, xe=xe, alpha_e=al, sigma_e=sg, alpha_t=al, sigma_t=sg, state_dtype=sdtype,
                 guidance_b=raw.guidance_b, per_sample=raw.e_cond.numel() // raw.e_cond.shape[0], coef_dev=coef_dev)
    if raw.param == PARAM_EDM:
        a.alpha_e, a.sigma_e = ns.conversion_words(al, sg, True)
    a.apg_words = be.apg_words(a, eta, norm_threshold, momentum, r_prev, r_out)
    a.apg_r = r_out
    return a


def _fdg_scales(fdg_scales):
    """model_wrapper's fdg_scales -> (levels, shared, tensor): the N shared scales as python floats, each rounded to
    fp32 once (a list or tuple of numbers), or None and the tensor `WrappedModel.fdg_args` converts once per (tensor,
    version, device, B) or reads in place (a 1-D tensor, a [B, N] tensor, or a list or tuple holding tensors, kept as a
    tuple and stacked on their device). The host never reads a tensor's values."""
    s = fdg_scales
    if isinstance(s, (list, tuple)) and any(torch.is_tensor(v) for v in s):
        if any(not torch.is_tensor(v) or v.numel() != 1 for v in s) or len({v.device for v in s}) != 1:
            raise ValueError("fdg_scales as a list or tuple of tensors takes N one-element tensors on one device")
        if any(v.is_complex() for v in s):
            raise ValueError("fdg_scales must be real, got {}".format(next(v.dtype for v in s if v.is_complex())))
        # the tensors themselves, not a stacked copy: fdg_args restacks them after an in-place write to any of them
        levels, shared, s = len(s), False, tuple(s)
    elif torch.is_tensor(s):
        if s.dim() not in (1, 2):
            raise ValueError("fdg_scales must be a list, a tuple, a 1-D tensor of N scales or a [B, N] tensor, got "
                             "shape {}".format(tuple(s.shape)))
        if s.is_complex():
            raise ValueError("fdg_scales must be real, got {}".format(s.dtype))
        levels, shared = s.shape[-1], False
    elif isinstance(s, (list, tuple)):
        if any(isinstance(v, (list, tuple)) for v in s):
            raise ValueError("fdg_scales as a list or tuple takes N numbers")
        levels, shared = len(s), True
    else:
        raise ValueError("fdg_scales must be a list, a tuple, a 1-D tensor of N scales or a [B, N] tensor, got "
                         "{!r}".format(type(s).__name__))
    if not 1 <= levels <= ops._lib.FDG_MAX_LEVELS:
        raise ValueError("fdg_scales takes 1 to {} levels, got {}".format(ops._lib.FDG_MAX_LEVELS, levels))
    if shared:
        return levels, tuple(torch.tensor([float(v) for v in s], dtype=torch.float32).tolist()), None
    return levels, None, s


def _fdg_output(be, raw: RawOutput) -> RawOutput:
    """A frequency-decoupled guidance evaluation as one network output: g in the outputs' dtype (1 launch), which the
    parameterisation then converts as it converts a single output."""
    fn = getattr(be, "fdg_guided", None)
    if fn is None:
        raise RuntimeError("fdg_scales needs an executor with fdg_guided; {} has none".format(
            getattr(be, "name", type(be).__name__)))
    return RawOutput(fn(raw.e_cond, raw.e_uncond, *raw.fdg), None, raw.param, 1.0)


def _scale_vector(guidance_scale, guidance_type):
    """model_wrapper's guidance_scale as per-sample scales (a 1-D tensor, or None for one scale). A python number, a
    0-dim or a one-element tensor is one scale, as before; any other tensor must be 1-D."""
    s = guidance_scale
    if not torch.is_tensor(s) or s.numel() == 1:
        return None
    if s.dim() != 1:
        raise ValueError("a per-sample guidance_scale must be 1-D, got shape {}".format(tuple(s.shape)))
    if guidance_type == "classifier":
        raise ValueError("a per-sample guidance_scale needs guidance_type='classifier-free'")
    return s


class WrappedModel:
    """Callable returned by `model_wrapper`: `model_fn(x, t_continuous) -> noise` (:309-330).

    Calling it reproduces the reference semantics. `DPM_Solver` additionally uses `raw()` to get
    the un-combined network outputs so that parameterisation + CFG are fused into the solver step.
    """

    def __init__(self, model, noise_schedule, model_type, model_kwargs, guidance_type, condition,
                 unconditional_condition, guidance_scale, classifier_fn, classifier_kwargs, guidance_rescale=0.,
                 apg_eta=None, apg_norm_threshold=0., apg_momentum=0., cfg_zero_star=False, cfg_zero_init_steps=0,
                 cfg_pp=False, guidance_mask=None, tcfg=False, fdg_scales=None, perp_neg=False):
        self.model = model
        self.cfg_pp = cfg_pp
        self.tcfg = tcfg
        self.perp_neg = perp_neg
        # frequency-decoupled guidance: its number of levels (0: off), shared scales or the per-sample tensor
        self.fdg_levels, self._fdg_shared, self._fdg_vec = (0, None, None) if fdg_scales is None else \
            _fdg_scales(fdg_scales)
        self._fdg_dev = None
        self.guidance_rescale = guidance_rescale
        self.cfg_zero_star = bool(cfg_zero_star)
        self.cfg_zero_init_steps = cfg_zero_init_steps
        self.apg_eta = apg_eta
        self.apg = None if apg_eta is None else (float(apg_eta), float(apg_norm_threshold), float(apg_momentum))
        self.noise_schedule = noise_schedule
        self.model_type = model_type
        self.model_kwargs = model_kwargs
        self.guidance_type = guidance_type
        self.cond_scales = None     # K >= 2 conditions (any K with masks): their K scales (python floats, fp32-rounded)
        # regional guidance: one _CondMask or None per condition (model_wrapper's guidance_mask, normalised to a list)
        self.cond_masks = None if guidance_mask is None else tuple(
            None if m is None else _CondMask(m) for m in guidance_mask)
        if guidance_type == "classifier-free" and isinstance(condition, (list, tuple)):
            condition, guidance_scale, self.cond_scales = _multi_condition(
                condition, unconditional_condition, guidance_scale, self.cond_masks is not None)
        self.condition = condition
        self.unconditional_condition = unconditional_condition
        if isinstance(guidance_scale, (list, tuple)) and self.cond_scales is None:
            guidance_scale = torch.tensor(list(guidance_scale), dtype=torch.float32)   # each value rounded once
        self.guidance_scale = guidance_scale
        self.classifier_fn = classifier_fn
        self.classifier_kwargs = classifier_kwargs
        self._c_in = None
        self._scale_vec = None if self.cond_scales is not None else _scale_vector(guidance_scale, guidance_type)
        self._gs = None
        self._gs1 = None

    # -- pieces of the reference closure ----------------------------------------------------
    def get_model_input_time(self, t_continuous):
        """[1/N, 1] -> [0, 1000*(N-1)/N] for discrete-time models (:271-280)."""
        if self.noise_schedule.schedule == 'discrete':
            return (t_continuous - 1. / self.noise_schedule.total_N) * 1000.
        if self.noise_schedule.schedule in ('flow', 'edm'):
            return self.noise_schedule.model_input_time(t_continuous)     # time_scale * sigma_t, or ln(s)/4
        return t_continuous

    def _call_model(self, x, t_continuous, cond=None, t_input=None):
        if t_input is None:
            t_input = self.get_model_input_time(t_continuous)
        if cond is None:
            return self.model(x, t_input, **self.model_kwargs)
        return self.model(x, t_input, cond, **self.model_kwargs)

    @property
    def per_sample_guidance(self) -> bool:
        """True when classifier-free guidance runs with one scale per sample (other guidance types ignore the scale)."""
        return self._scale_vec is not None and self.guidance_type == "classifier-free"

    @property
    def n_cond(self) -> int:
        """Number of conditions of a multi-condition run (K >= 2, or K >= 1 with guidance masks), else 0."""
        return 0 if self.cond_scales is None else len(self.cond_scales)

    def guidance_options(self) -> frozenset:
        """The guidance options (keys of _OPTIONS) the wrapper's attributes select now."""
        if self.guidance_type != "classifier-free":
            return frozenset()
        return frozenset(k for k, on in (
            ("several", self.n_cond >= 2), ("mask", self.cond_masks is not None), ("perp", self.perp_neg),
            ("rescale", self.guidance_rescale != 0), ("apg", self.apg is not None), ("cfgzero", self.cfg_zero_star),
            ("cfgpp", self.cfg_pp), ("tcfg", self.tcfg), ("fdg", self.fdg_levels > 0),
            ("per_sample", self._scale_vec is not None), ("zero_init", self.cfg_zero_init_steps > 0),
            ("momentum", self.apg is not None and self.apg[2] != 0)) if on)

    def _form(self, plain: bool) -> tuple:
        """(form, host constants) of a guided evaluation of the two halves, as the wrapper's attributes select it now
        (`plain`: the plain guided noise of a direct call, never CFG++)."""
        if self.apg is not None:
            return "apg", self.apg
        if self.cfg_zero_star:
            return "cfgzero", ()
        if self.cfg_pp and not plain:
            return "cfgpp", ()
        if self.tcfg:
            return "tcfg", ()
        if self.guidance_rescale != 0:
            return "rescale", (self.guidance_rescale,)
        return "", ()

    def _one_scale(self):
        """The single guidance scale as the host reads it. A 0-dim or one-element tensor is read once per (tensor,
        version), not at every evaluation: on the device that read is a host synchronisation, which a steady-state
        loop must not pay and a graph capture cannot contain."""
        s = self.guidance_scale
        if not torch.is_tensor(s):
            return s
        key = (id(s), s._version)
        if self._gs1 is None or self._gs1[0] != key:
            self._gs1 = (key, float(s), s)          # (the tensor is kept alive so that its id cannot be recycled)
        return self._gs1[1]

    @property
    def uses_cfg(self) -> bool:
        # (several conditions: guidance_scale is their tuple of scales, never equal to 1 -- always combined, no bypass)
        # (CFG++ reads both halves at every evaluation: a scalar scale of 1 is combined, not bypassed)
        # (frequency-decoupled guidance always combines both halves, whatever its scales)
        return self._combines() or self.cfg_pp or self.fdg_levels > 0

    def _combines(self) -> bool:
        """The plain guided noise combines the two halves (the reference's test :323)."""
        return (self.guidance_type == "classifier-free" and self.unconditional_condition is not None
                and (self._scale_vec is not None or self._one_scale() != 1.))

    def input_copies(self) -> int:
        """How many copies of x the network input holds: K + 1 with K >= 2 conditions, 2 under CFG (:326), else 1."""
        if self.cond_scales is not None:
            return len(self.cond_scales) + 1
        return 2 if self.uses_cfg else 1

    def _scales(self, x) -> torch.Tensor:
        """The per-sample scales as the kernels read them: fp32 [B] on x's device. A contiguous fp32 tensor already
        there is read in place (so values written into it between graph replays take effect); any other form is
        converted once per (tensor, version, device). Never reads the values on the host."""
        s = self._scale_vec
        if s.numel() != x.shape[0]:
            raise ValueError("guidance_scale has {} values for a batch of {}".format(s.numel(), x.shape[0]))
        if s.device == x.device and s.dtype == torch.float32 and s.is_contiguous():
            return s
        key = (id(s), s._version, str(x.device))
        if self._gs is None or self._gs[0] != key:
            # the source is kept alive next to the key so that its id cannot be recycled
            self._gs = (key, s.detach().to(device=x.device, dtype=torch.float32).contiguous(), s)
        return self._gs[1]

    def fdg_args(self, x) -> tuple:
        """(scales, levels) of a frequency-decoupled guidance evaluation at x: the shared python floats, or fp32
        [B, N] on x's device. A contiguous fp32 [B, N] tensor already there is read in place (values written into it
        between graph replays take effect); any other form is converted once per (tensor, version, device, B). Checks
        x against the size rule, and the per-sample rows against x's batch (ValueError); never reads device values on
        the host."""
        L = self.fdg_levels
        ops.fdg_check(x.shape, L)
        if self._fdg_shared is not None:
            return self._fdg_shared, L
        s, B = self._fdg_vec, x.shape[0]
        listed = isinstance(s, tuple)            # N one-element tensors
        if not listed and s.dim() == 2:
            if s.shape[0] != B:
                raise ValueError("fdg_scales has {} rows for a batch of {}".format(s.shape[0], B))
            if s.device == x.device and s.dtype == torch.float32 and s.is_contiguous():
                return s, L
        key = (tuple((id(v), v._version) for v in (s if listed else (s,))), str(x.device), B)
        if self._fdg_dev is None or self._fdg_dev[0] != key:
            # the source is kept alive next to the key so that its id cannot be recycled
            v = torch.stack([t.detach().reshape(()) for t in s]) if listed else s.detach()
            v = v.to(device=x.device, dtype=torch.float32)
            self._fdg_dev = (key, v.expand(B, L).contiguous(), s)
        return self._fdg_dev[1], L

    @property
    def fusable(self) -> bool:
        """False only for classifier guidance (needs autograd through the user's classifier)."""
        return self.guidance_type != "classifier"

    def input_rows(self, batch: int) -> int:
        """Length of the time vector the network receives for a batch (doubled under CFG :327, (K+1)-fold with K >= 2
        conditions)."""
        return self.input_copies() * batch

    def _cond_in(self):
        """cat([unconditional_condition, condition]) (:328), or cat([uc, c1, ..., cK]) with several conditions;
        constant over a run, so built once."""
        uc, c = self.unconditional_condition, self.condition
        if self.cond_scales is not None:
            key = tuple((id(v), getattr(v, "_version", 0)) for v in (uc,) + c)
            if self._c_in is None or self._c_in[0] != key:
                self._c_in = (key, torch.cat([uc, *c]), (uc, c))
            return self._c_in[1]
        key = (id(uc), getattr(uc, "_version", 0), id(c), getattr(c, "_version", 0))
        if self._c_in is None or self._c_in[0] != key:
            # the pair is kept alive next to the key so that neither id can be recycled
            self._c_in = (key, torch.cat([uc, c]), (uc, c))
        return self._c_in[1]

    def raw(self, x, t_continuous, t_input=None, x_in=None, plain=False) -> RawOutput:
        """Run the network exactly as the reference does, return its un-combined output(s).

        `t_input`, when given, is the precomputed model-input time vector (`input_rows(B)` long,
        same values as get_model_input_time would produce) so that no per-call arithmetic runs.
        `plain`: the outputs of the plain guided noise (a direct call of this callable), never marked for CFG++."""
        param = PARAM_BY_NAME[self.model_type]
        if self.guidance_type == "uncond":
            return RawOutput(self._call_model(x, t_continuous, t_input=t_input), None, param, 1.0)
        if self.guidance_type == "classifier-free" and self.cond_scales is not None:
            n = len(self.cond_scales) + 1
            for m in self.cond_masks or ():
                if m is not None:
                    m.check(x.shape)                              # (before any launch)
            if x_in is None:
                x_in = ops.backend().replicate(x, n)              # cat([x] * (K+1)) (the solver hands over a prebuilt one)
            t_in = None if t_input is not None else torch.cat([t_continuous] * n)
            outs = self._call_model(x_in, t_in, cond=self._cond_in(), t_input=t_input).chunk(n)   # uncond first
            return RawOutput(outs[1], outs[0], param, 1.0, e_conds=tuple(outs[1:]), scales=self.cond_scales,
                             masks=self.cond_masks, form="perp" if self.perp_neg else "")
        if self.guidance_type == "classifier-free":
            gb = self._scales(x) if self._scale_vec is not None else None     # (checked before the network runs)
            fdg = self.fdg_args(x) if self.fdg_levels else None               # likewise
            if not ((self._combines() or self.fdg_levels > 0) if plain else self.uses_cfg):
                return RawOutput(self._call_model(x, t_continuous, cond=self.condition, t_input=t_input), None, param, 1.0)
            if x_in is None:
                x_in = ops.backend().duplicate(x)              # cat([x] * 2) :326 (the solver hands over a prebuilt one)
            t_in = None if t_input is not None else torch.cat([t_continuous] * 2)
            out_u, out_c = self._call_model(x_in, t_in, cond=self._cond_in(), t_input=t_input).chunk(2)  # uncond first
            if fdg is not None:
                return RawOutput(out_c, out_u, param, 1.0, form="fdg", fdg=fdg)
            form, consts = self._form(plain)
            return RawOutput(out_c, out_u, param, 1.0 if gb is not None else float(self._one_scale()), gb, form=form,
                             consts=consts)
        raise RuntimeError("raw() is not available with classifier guidance")

    def _alpha_sigma(self, t_continuous):
        """Host scalars [(alpha_t, sigma_t)]: one pair when all labels of the batch are equal (the solver's
        case), else one pair per sample (model_fn called directly with a vector of different times)."""
        tc = t_continuous.detach().reshape(-1).cpu()
        ns = self.noise_schedule
        if tc.numel() > 1 and not bool((tc == tc[0]).all()):
            return list(zip(ns.marginal_alpha(tc).tolist(), ns.marginal_std(tc).tolist()))
        t0 = tc[:1]
        return [(float(ns.marginal_alpha(t0)), float(ns.marginal_std(t0)))]

    @staticmethod
    def _per_sample(pairs, batch, launch):
        """Run `launch(rows, alpha, sigma)` once for the whole batch, or once per sample when the time labels
        differ (alpha_t, sigma_t are launch constants of the kernels)."""
        if len(pairs) == 1:
            return launch(slice(None), *pairs[0])
        assert len(pairs) == batch, "one time label per sample expected"
        return torch.cat([launch(slice(i, i + 1), al, sg) for i, (al, sg) in enumerate(pairs)])

    def __call__(self, x, t_continuous):
        be = ops.backend()
        if self.guidance_type == "classifier":
            assert self.classifier_fn is not None
            t_input = self.get_model_input_time(t_continuous)
            with torch.enable_grad():
                x_in = x.detach().requires_grad_(True)
                log_prob = self.classifier_fn(x_in, t_input, self.condition, **self.classifier_kwargs)
                cond_grad = torch.autograd.grad(log_prob.sum(), x_in)[0]
            pairs = self._alpha_sigma(t_continuous)
            out = self._call_model(x, t_continuous)
            param = PARAM_BY_NAME[self.model_type]
            xo, grad = x.to(out.dtype), cond_grad.to(out.dtype)

            def guided(rows, alpha, sigma):
                o = out[rows]
                if param != PARAM_NOISE:
                    o = be.step(StepArgs(form=FORM_NONE, n_model=1, e_cond=o, xe=xo[rows], param=param,
                                         alpha_e=alpha, sigma_e=sigma, state_dtype=out.dtype))[0]
                # noise - guidance_scale * sigma_t * cond_grad (:321); (s*sigma) is formed in fp32 first
                gs = float(torch.tensor(sigma, dtype=torch.float32) * self.guidance_scale)
                return ops.lincomb(o, [grad[rows]], 1.0, [-gs])
            return self._per_sample(pairs, x.shape[0], guided)
        r = self.raw(x, t_continuous, plain=True)
        if r.form == "fdg":
            r = _fdg_output(be, r)        # g, then converted as one network output
        if r.form == "perp":
            r = _perp_output(be, r)       # over the whole batch: each sample's word reads its own values only
        if r.e_uncond is None and r.param == PARAM_NOISE:
            return r.e_cond
        if r.form == "apg":
            # adaptive projected guidance: the words pass, then the guided x0 converted to noise (a direct call is the
            # first evaluation of its own: no momentum)
            xo = x.to(r.e_cond.dtype)

            def apg(rows, alpha, sigma):
                rr = dataclasses.replace(r, e_cond=r.e_cond[rows], e_uncond=r.e_uncond[rows],
                                         guidance_b=None if r.guidance_b is None else r.guidance_b[rows])
                a = _apg_args(be, rr, xo[rows], (alpha, sigma), r.e_cond.dtype, False, self.noise_schedule)
                a.form = FORM_NONE
                return be.step(a)[0]
            return self._per_sample(self._alpha_sigma(t_continuous), x.shape[0], apg)
        pairs = self._alpha_sigma(t_continuous) if r.param != PARAM_NOISE else [(1.0, 0.0)]
        if r.param == PARAM_EDM:
            pairs = [self.noise_schedule.conversion_words(al, sg, False) for al, sg in pairs]   # eps words
        needs_x = r.param in (PARAM_BY_NAME["x_start"], PARAM_BY_NAME["v"], PARAM_FLOW, PARAM_EDM)
        xo = x.to(r.e_cond.dtype) if needs_x else None
        words = _words(be, r)          # over the whole batch: each sample's words read its own values only

        def convert(rows, alpha, sigma):
            a = StepArgs(form=FORM_NONE, n_model=2 if r.e_uncond is not None else 1, e_cond=r.e_cond[rows],
                         e_uncond=None if r.e_uncond is None else r.e_uncond[rows], param=r.param,
                         guidance=r.guidance, alpha_e=alpha, sigma_e=sigma, state_dtype=r.e_cond.dtype)
            _guidance_args(a, words, r, rows)
            if needs_x:
                a.xe = xo[rows]
            return be.step(a)[0]
        return self._per_sample(pairs, x.shape[0], convert)


def model_wrapper(model, noise_schedule, model_type="noise", model_kwargs={}, guidance_type="uncond",
                  condition=None, unconditional_condition=None, guidance_scale=1., classifier_fn=None,
                  classifier_kwargs={}, guidance_rescale=0., apg_eta=None, apg_norm_threshold=0., apg_momentum=0.,
                  cfg_zero_star=False, cfg_zero_init_steps=0, cfg_pp=False, guidance_mask=None, tcfg=False,
                  fdg_scales=None, perp_neg=False):
    """Wrap a network into `model_fn(x, t_continuous) -> noise`; same contract as the reference
    (:170-334): model_type in {noise, x_start, v, score}, guidance_type in {uncond, classifier,
    classifier-free}.

    model_type="flow" (not in the reference; needs a `NoiseScheduleFlow`): the network predicts the velocity
    v = eps - x0 of a flow-matching model. The solver converts it straight into its own space, x0 = x - sigma_t*v for
    dpmsolver++ and eps = x + alpha_t*v for dpmsolver (this callable returns the latter), two rounded ops and no
    division. Under classifier-free guidance in any form each output is converted first and the converted values are
    combined; guidance_rescale combines and rescales the raw velocities, then converts. A NoiseScheduleFlow also takes
    "noise" and "x_start" networks; "v" and "score" (VP formulas) and guidance_type="classifier" are rejected.

    model_type="edm" (not in the reference; needs a `NoiseScheduleEDM`, which takes no other model type): the network
    is the raw F of an EDM-preconditioned model and receives the solver's state y = c_in*x and c_noise = ln(s)/4. The
    solver converts F straight into its own space with two words computed on the host from the fp32 marginals and
    rounded once: x0 = (sd^2*alpha_t)*y + (sd*sigma_t)*F for dpmsolver++ and denoise_to_zero, eps = sigma_t*y -
    (sd*alpha_t)*F for dpmsolver (this callable returns the latter), three rounded ops and no division. Guidance works
    as for "flow"; guidance_type="classifier" and DPM_Solver(reference_rounding=True) are rejected.

    guidance_rescale=phi (classifier-free guidance only; not in the reference): guidance rescale of Lin et al.
    2023 as diffusers' `rescale_noise_cfg` does it, in the network's output space (eps for a noise network, v for
    a v network): g = out_u + s*(out_c - out_u), r_b = std(out_c_b)/std(g_b) per sample (unbiased),
    g' = phi*(g*r_b) + (1 - phi)*g, then the parameterisation converts g'. It applies only when the combine
    runs (scale != 1 and an unconditional condition); 0 (default) is plain CFG.

    guidance_scale (classifier-free guidance) may also hold one scale per sample of x: a 1-D tensor, list or tuple of
    B numbers (not in the reference). Row b of every result is then that of the same call with
    guidance_scale=float(s[b]), each scale rounded to fp32 once; a row with s[b] == 1 gets the conditional output alone,
    as the reference's bypass does, although the network still sees the doubled batch. A contiguous fp32 tensor on
    x's device is read in place by the kernels (a captured graph sees values written into it); other forms are
    converted once and cached. A python number, a 0-dim or a one-element tensor is one scale, as before; such a tensor is
    read on the host once per (tensor, version), so a steady-state loop does not synchronise on it.

    condition (classifier-free guidance) may also be a list or tuple of K conditions, 1 <= K <= 4 (composable prompts,
    Liu et al. 2022; not in the reference, whose cat([uc, c]) refuses a list). guidance_scale then holds exactly K
    scales (a list, tuple or 1-D tensor), read on the host once here and rounded to fp32 once. The network runs once
    per evaluation on cat([x] * (K+1)) with cat([uc, c1, ..., cK]); every output block is converted by the
    parameterisation, then eps = eps_u + s1*(eps_1 - eps_u) + ... + sK*(eps_K - eps_u), left to right in fp32, as
    torch's eager ops compute it. Every output is combined, whatever the scales (no bypass). One condition in a list is
    exactly the tensor form. With K >= 2: unconditional_condition is required, and guidance_rescale, per-sample scales
    and DPM_Solver(reference_rounding=True) are not available (ValueError).

    apg_eta=eta (classifier-free guidance only; not in the reference; None, the default, is off): adaptive projected
    guidance (Sadat, Hilliges and Weber, ICLR 2025) on the denoised prediction. Both outputs are converted to x0 by the
    parameterisation, c = x0_cond and D = c - x0_uncond; with apg_momentum=beta != 0, R = D + beta*R_prev across the
    evaluations of one sample() / inverse() run (R = D at its first evaluation and in a direct call of this callable);
    with apg_norm_threshold=r > 0, k = min(1, r/||R||) per sample, else 1; p = <R, c>/max(||c||, 1e-12)^2 per sample;
    guided x0 = c + (w - 1)*(k*R - (1 - eta)*k*p*c). The guided x0 is then what the solver buffers (dpmsolver++,
    thresholded when enabled) or converts to noise with the x_start conversion (dpmsolver, and this callable). eta = 1,
    r = 0, beta = 0 is plain CFG in exact arithmetic. It takes a scalar or a per-sample guidance_scale; a scalar scale of
    1 keeps the bypass (one network half, no APG), a per-sample scale of 1 gives that row c. Not available (ValueError):
    other guidance types, no unconditional_condition, several conditions, guidance_rescale != 0, a non-finite eta or
    momentum, a negative or non-finite threshold, DPM_Solver(reference_rounding=True) and apg_momentum != 0 with
    method="adaptive".

    cfg_zero_star=True (classifier-free guidance only; not in the reference; default False): CFG-Zero* (Fan, Zheng,
    Yeh and Liu 2025, arXiv:2503.18886), in the network's raw output space -- the velocity of a "flow" network, the
    noise of a "noise" one, whatever the network returns for "x_start", "v", "score" and "edm". Per sample b, with c
    and u the conditional and unconditional outputs flattened over all non-batch dimensions in storage order:
        s*_b = fl32(<c_b, u_b> / (||u_b||^2 + 1e-8))   (the sums in fp64 over the fp32-widened outputs, the division in
                                                       fp64, rounded to fp32 once; 1e-8 is diffusers' epsilon)
        us = u*s*_b;  g = us + w_b*(c - us)             (three fp32 ops, each rounded, no contraction, in this order)
    and the parameterisation then converts g as it converts a single output (combine raw, convert the result, as
    guidance_rescale does). diffusers casts s* to the model's dtype and combines in it (bf16 for a bf16 network); this
    library combines in fp32, as its plain CFG combine does. A scalar guidance_scale of 1 keeps the bypass (one network
    half, the conditional output alone); a per-sample scale of 1 gives that row c.
    cfg_zero_init_steps=K (an int >= 0; needs cfg_zero_star=True): zero-init. The first K network evaluations of each
    sample() / inverse() run (DPM_Solver and UniPC) have a raw output of exactly 0 and do not call the network; the
    solver then takes a one-output step on that 0 (for "flow" x0 = x exactly). Evaluations are counted in run order:
    one per step for multistep and UniPC, every intermediate evaluation for singlestep, and the denoise_to_zero
    evaluation. A direct call of this callable is never zeroed. Not available (ValueError): other guidance types, no
    unconditional_condition, several conditions, guidance_rescale != 0, apg_eta, DPM_Solver(reference_rounding=True),
    a cfg_zero_init_steps that is not an int >= 0 or that is set without cfg_zero_star=True, and cfg_zero_init_steps
    > 0 with method="adaptive" (rejected steps leave "the first K evaluations" undefined).

    cfg_pp=True (classifier-free guidance only; not in the reference; default False): CFG++ (Chung, Kim, Park, Nam and
    Ye, ICLR 2025, arXiv:2406.08070). It changes the solver update, not the guided value: each update denoises with the
    guided x0 and re-noises with the UNCONDITIONAL noise, so that the DDIM step is x_t = alpha_t*x0_g + sigma_t*eps_u.
    Scales are those of CFG++ (about 0.2 to 1), not those of plain CFG (about 5 to 12); guidance_scale is a scalar or a
    per-sample [B] tensor as above. DPM_Solver(fn, ns, algorithm_type="dpmsolver++").sample(x, method="multistep",
    order=1 or 2, ...) then computes, at every evaluation, for every element, in fp32 with each op rounded and no
    contraction (S = the state dtype):
        U = round_S(T_u)   T_u: the x0 the unguided step buffers for the unconditional output alone (every
                           parameterisation as without guidance)
        G = round_S(T_g)   T_g: the x0 the classifier-free step buffers with this sample's scale (a per-sample scale of 1
                           takes the conditional output; a scalar scale of 1 is combined, not bypassed: CFG++ always
                           needs both halves)
        d = G - U
        order 1 (first-update coefficients a, c0):        x_t = (a*x + c0*U) + g*d
        order 2 (multistep coefficients a, c0, c1, w0):   x_t = ((a*x + c0*U) + g*d) + c1*(w0*(G - U_prev))
    with g = alpha_t, the fp32 alpha of the update's end time that c0 is formed from, and U_prev the previous update's U:
    the multistep buffer holds U, not G. In exact arithmetic order 1 is alpha_t*G + sigma_t*eps_u, the paper's DDIM
    CFG++, and order 2 the 2M CFG++ recurrence; in VE coordinates (x^ = x/alpha, lambda = -log(sigma/alpha), h the
    step in lambda, r the ratio of the previous step to h):
        x^' = G + e^-h*(x^ - U) - expm1(-h)/(2r)*(G - U_prev)       (solver_type="taylor": its c1, by the same rule)
    A network blind to the condition (e_c == e_u) gives d = 0, and a CFG++ run then equals the plain DPM-Solver++ run at
    any scale. denoise_to_zero returns G; a direct call of this callable returns the plain guided noise. Accepted:
    sample() and inverse() with every skip type, lower_order_final, return_intermediate, correcting_xt_fn, capture()
    and batch sharding, on every schedule and model type. Not available (ValueError before any launch): other guidance
    types, no unconditional_condition, several conditions, guidance_rescale != 0, apg_eta, cfg_zero_star, a cfg_pp
    that is not a bool, and in the solver algorithm_type="dpmsolver", order 3, singlestep, singlestep_fixed and adaptive
    methods, UniPC, the direct update methods (dpm_solver_first_update, multistep_dpm_solver_*_update, ...), dynamic
    thresholding and any correcting_x0_fn, and reference_rounding=True.

    guidance_mask=m or [m1, ..., mK] (classifier-free guidance only; not in the reference; None, the default, changes
    nothing): regional guidance, one weight mask per condition of condition=c or [c1, ..., cK] (K = 1 to 4), for
    regional prompting and MultiDiffusion-style region composition (Bar-Tal et al. 2023). Each entry is a tensor or None
    (all ones). A mask broadcasts to x's shape [B, C, *spatial] by torch's rules -- [H, W], [1, 1, H, W], [B, 1, H, W],
    [B, C, H, W], [B, 1, 1, 1] (one weight per sample and condition), ... -- so its batch extent is 1 or B; this is
    checked against x at the first evaluation and rejected (ValueError) before any launch. Values are taken as given in
    fp32 (bool is 0/1); nothing checks them on the device and nothing synchronises. The network runs on all K+1 blocks,
    as with several conditions (masks skip no network work). Per element i, in the network's output space after the
    parameterisation converts each block, in fp32 with each op rounded and no contraction:
        eps = eps_u;  for k = 1..K:  w = fl32(s_k)*m_k(i);  eps = eps + w*(eps_k - eps_u)
    then eps -> x0, the thresholding clamp and the update as with several conditions. No term is bypassed: a zero
    weight still evaluates 0*(eps_k - eps_u) (NaN where that difference is infinite, as a zero scale does). Masks of
    ones give w == s_k, so the run equals the unmasked multi-condition run bit for bit for K >= 2, and for K = 1 the
    one-condition CFG run when s != 1 (at s == 1 that run bypasses; this one combines). With masks that sum to 1 at
    every element and one shared scale s, the result is, in exact arithmetic, ordinary CFG with scale s applied to the
    mask-weighted average of the conditional outputs: the recipe for "average the regions". A contiguous fp32 mask on
    x's device that already has its weight map's layout ([H, W] or [B, 1, H, W] for a row-major x, [B, 1, 1, 1], or a
    [B, C, H, W] mask laid out like x) is read in place, so a captured graph sees values written into it; other masks
    are converted once per (tensor, version, x shape, x memory format). guidance_scale is s or [s1, ..., sK] (one
    python float or one-element tensor per condition). Accepted: everything several conditions accept -- every model
    type and schedule, both algorithms, singlestep, multistep, singlestep_fixed, adaptive (host or device controller),
    dynamic thresholding, denoise_to_zero, inverse(), return_intermediate, capture() and batch sharding (each rank
    passes the masks of its own rows); a direct call of this callable returns the masked combine. Not available
    (ValueError): other guidance types, no unconditional_condition, a mask count other than K, an entry that is neither
    a tensor nor None, a per-sample guidance_scale (use a [B, 1, 1, 1] mask), guidance_rescale != 0, apg_eta,
    cfg_zero_star, cfg_pp, UniPC and DPM_Solver(reference_rounding=True).

    tcfg=True (classifier-free guidance only; not in the reference; default False; anything other than a bool is a
    ValueError): tangential-damping CFG ("TCFG: Tangential Damping Classifier-free Guidance", CVPR 2025; diffusers'
    TangentialClassifierFreeGuidance guider, ComfyUI's TCFG node). The damping works in the network's raw output space,
    as cfg_zero_star does: the noise of a "noise" network, the velocity of a "flow" one, whatever the network returns
    for "x_start", "v", "score" and "edm" -- the space of diffusers' guider. ComfyUI damps x - denoised, which is
    sigma*eps or sigma*v for noise and flow networks; the damping is invariant to a per-sample factor common to both
    outputs, so it gives the same words there.
    Definition: per sample b, with c and u the conditional and unconditional outputs flattened over all non-batch
    dimensions in storage order, M the 2 x D matrix with rows u and c and v1 its first right singular vector, the damped
    unconditional output is u' = <u, v1>*v1 (diffusers and ComfyUI compute it with torch.linalg.svd), and the guided
    raw output g = u' + w_b*(c - u') is then converted by the parameterisation as it converts a single output.
    This library evaluates u' in closed form from the 2 x 2 Gram matrix, u' = wu_b*u + wc_b*c. A = ||u||^2,
    B = <u, c>, C = ||c||^2 are fp64 sums of the fp32-widened outputs, in the chunking, thread ownership and chunk-merge
    order of the CFG-Zero* pass, so the words of sample b depend on sample b's values only. Then, in fp64 with each
    operation rounded:
        h = 0.5*(A - C);  r = sqrt(h*h + B*B)
        if C >= A:  p = B;      q = (-h) + r
        else:       p = h + r;  q = B
        pp = p*p;  n2 = pp + q*q
        wu = fl32(pp / n2);  wc = fl32((p*q) / n2)
    (p, q) is the top eigenvector of the Gram matrix, taken from the row without cancellation, and the closed form is
    the eigen identity. n2 == 0 happens only when A == C and B == 0 (both outputs zero included): the top singular
    direction is then not unique and the words are (1, 0), plain CFG. A sum that is not finite gives NaN words. Then
    per element, in fp32 with each operation rounded and no contraction, in this order:
        us = u*wu + c*wc;   g = us + w*(c - us);   value = convert(g)
    diffusers casts u' to the model's dtype and combines in it; this library combines in fp32, as cfg_zero_star and
    plain CFG do. Consequences: a network blind to the condition (c == u) gives A = B = C, r = |B| exactly and the
    words exactly (0.5, 0.5), so us == u and g == u for normal operands: such a run equals the unguided run by value,
    at any scale and in every state dtype. Rank-1 pairs (c = k*u) give u' = u in exact arithmetic, plain CFG. A scalar
    guidance_scale of 1 keeps the bypass (one network half, the conditional output alone, no words pass); a per-sample
    scale of 1 gives that row c. Cost per guided evaluation: the words pass (2 launches reading both halves once) and
    the fused step; with dynamic thresholding, and under UniPC, g is materialised once in fp32 (+1 launch) first.
    Accepted: scalar or per-sample [B] scales, every model type and schedule (VP discrete, linear and cosine, flow,
    EDM), both algorithms, singlestep, multistep, singlestep_fixed and adaptive (host or device controller), dynamic
    thresholding, correcting_x0_fn / correcting_xt_fn, denoise_to_zero, inverse(), return_intermediate, capture(),
    batch sharding (the words are per sample: no collective) and UniPC. A direct call of this callable returns the
    converted TCFG value. Not available (ValueError before any launch and any network call): other guidance types, no
    unconditional_condition, several conditions, guidance_mask, guidance_rescale != 0, apg_eta, cfg_zero_star, cfg_pp
    and DPM_Solver(reference_rounding=True).

    perp_neg=True (classifier-free guidance with condition=[c_1, ..., c_K], 2 <= K <= 4; not in the reference; default
    False; anything other than a bool is a ValueError): perpendicular negative prompts (Perp-Neg; Armandpour,
    Sadeghian, Zheng, Sadeghian and Zhou, arXiv:2304.04968; ComfyUI's PerpNeg / PerpNegGuider). c_1 is the positive
    prompt; every later condition loses, per sample, its component along c_1's direction before it is weighted, so a
    negative prompt no longer removes part of what the positive one asks for. Negatives take negative scales, as they
    do with several conditions; ComfyUI's cond_scale s and neg_scale n are guidance_scale=[s, -s*n] with the empty
    prompt as unconditional_condition. With d_k = e_k - e_u the raw network outputs' differences, in exact arithmetic:
        eps = e_u + s_1*d_1 + sum_{k>=2} s_k*(d_k - (<d_k, d_1>/||d_1||^2)*d_1)
    The projection coefficient is taken in the network's raw output space, as cfg_zero_star and tcfg take theirs; every
    parameterisation converts the blocks of a sample by one affine map with a shared x term, so the ratio is the same
    in the converted space up to rounding. Exact arithmetic, per sample b, all values in storage order:
        N = sum d_1*d_1,  P_k = sum d_k*d_1 (k >= 2)     (fp64: each output widened, d_k = e_k - e_u in fp64, the sums
                                                         in the chunking and merge order of the CFG-Zero* pass)
        c_k = P_k / N, or 0 when N == 0 (condition 1 equals the unconditional output: the plain multi-condition combine)
        w_1 = fl32(s_1 - s_2*c_2 - ... - s_K*c_K)      (fp64 left to right, each op rounded, s_k = the fp32 scale)
    and a non-finite N or P_k gives a NaN w_1. The evaluation is then the regional-guidance one with the scales
    (1, s_2, ..., s_K) and w_1 as condition 1's one-weight-per-sample mask: eps = eps_u + w_1*(eps_1 - eps_u) +
    s_2*(eps_2 - eps_u) + ..., each block converted by the parameterisation first, every op rounded to fp32. The sums
    run per sample, not over the whole batch: rows stay independent and batch sharding needs no collective. ComfyUI
    normalises over the whole batch; for B = 1 the two agree. Consequences: negatives that differ from e_u only where
    c_1 does not give P_k = +0 and w_1 == s_1, the run without perp_neg bit for bit; a negative exactly parallel to
    the positive cancels its own effect to rounding; a condition-blind network gives the unguided run. Cost per guided
    evaluation: the words pass (2 launches, reading the K+1 outputs once, no host sync, so capture() replays it) and
    the masked fused step.
    Accepted: everything several conditions accept -- every model type and schedule, both algorithms, singlestep,
    multistep, singlestep_fixed, adaptive (host or device controller), dynamic thresholding, correcting_x0_fn /
    correcting_xt_fn, denoise_to_zero, inverse(), return_intermediate, capture() and batch sharding; a direct call of
    this callable returns the converted Perp-Neg value. Not available (ValueError before any launch and any network
    call): other guidance types, no unconditional_condition, fewer than two conditions, guidance_mask, and everything
    several conditions refuse (guidance_rescale, per-sample scales, apg_eta, cfg_zero_star, cfg_pp, tcfg, fdg_scales,
    UniPC and DPM_Solver(reference_rounding=True)). Not offered: per-sample Perp-Neg scales, Gram-Schmidt among the
    negatives (each is projected against the positive only), the paper's view-dependent weights for text-to-3D.

    fdg_scales=[w_0, ..., w_{N-1}] (classifier-free guidance only; not in the reference; default None: off):
    frequency-decoupled guidance (Sadat, Vontobel, Salehi and Weber, "Guidance in the Frequency Domain Enables
    High-Fidelity Sampling at Low CFG Scales", 2025; diffusers' FrequencyDecoupledGuidance guider). c - u is split into
    the N levels of a Laplacian pyramid over the last two dims (H, W) of x, and level l gets scale w_l: w_0 the finest
    (highest-frequency) level, w_{N-1} the coarsest, diffusers' order ([10.0, 5.0] is its default); 1 <= N <= 5.
    Accepted forms: a list or a tuple of N numbers or one-element tensors, or a 1-D tensor of N values (shared by the
    batch), or a [B, N] tensor with one row per sample. Numbers are rounded to fp32 once when the wrapper is built.
    A contiguous fp32 [B, N] tensor on x's device is read in place (a capture() replay sees values written into it);
    any other tensor form is converted on the device once per (tensor, version, device, B), so in-place writes to it
    take effect at the next evaluation. The host never reads a tensor's values. guidance_scale must stay at its default (fdg_scales replaces it); both halves are
    always combined, whatever the scales. The combine runs in the network's raw output space, as cfg_zero_star and tcfg
    do; every conversion is a per-sample affine map shared by both halves and the operator is linear in c - u, so the
    space does not change the result in exact arithmetic.
    Planes: every non-batch index other than the last two names one plane, so x needs at least 4 dims; H and W must each
    be divisible by 2^(N-1) with a quotient of at least 3, and H*W at most 16384 (128 x 128: SD 1.x/2.x latents are
    64 x 64, SDXL / SD3-size latents 128 x 128); the library states the rule once (dpm_fdg_supported). Violations raise
    ValueError against x before the network runs.
    Definition, per plane and sample, fp32 with each product rounded, sums left to right, no contraction, and
    delta_l = fl32(w_l - w_{l-1}):
        d = c - u;  G_0 = d;  G_{l+1} = Down(G_l)                        (l < N-1)
        E_{N-1} = delta_{N-1}*G_{N-1};  E_l = delta_l*G_l + Up(E_{l+1})  (l = N-2 .. 1)
        g = (u + w_0*d) + Up(E_1)   (N >= 2);   g = u + w_0*d   (N == 1)
    Down (n even -> n/2): out[i] = sum_k h_k*a[R(2i-2+k)], h = [1, 5, 10, 10, 5, 1]/32. Up (m -> 2m):
    out[2i] = (1*a[R(i-2)] + 21*a[R(i-1)] + 35*a[R(i)] + 7*a[R(i+1)])/64, out[2i+1] = (7*a[R(i-1)] + 35*a[R(i)] +
    21*a[R(i+1)] + 1*a[R(i+2)])/64, with the exact fp32 weights; R reflects without repeating the edge (R(j) = -j for
    j < 0, 2(n-1) - j for j > n-1). In 2-D both filters run along W on every row first, then along H. Down is the 5 x 5
    binomial blur with reflect borders followed by half-pixel bilinear 1/2 (kornia's pyrdown, as diffusers' guider uses
    it); Up is bilinear x2 followed by the blur in the interior and reflects on the coarse grid at the borders. In exact
    arithmetic this is diffusers' per-level form u_l + w_l*(c_l - u_l) on the pyramids of c and u, reconstructed; it
    needs one pyramid, of d only. Bit agreement with kornia is not claimed.
    g is stored in the network's output dtype and then converted by the parameterisation as a single output, so the
    update runs on the packet step kernels of that dtype pair. For 16-bit networks this rounds g once more, the size of
    the network output's own rounding. Consequences: N == 1 is the CFG combine u + w*(c - u) op for op (a noise network
    with fp32 outputs and w != 1 gives the plain CFG run bit for bit; at w == 1 plain CFG bypasses to c and this does
    not); equal scales give the N == 1 value (up to the sign of a zero); a condition-blind network (c == u) gives g = u,
    the unguided run, in every state dtype. Cost per guided evaluation: one pyramid launch (c and u read once, g written
    once), then the one-output step.
    Accepted: shared or [B, N] scales, every model type and schedule (VP discrete, linear and cosine, flow, EDM), both
    algorithms, singlestep, multistep, singlestep_fixed and adaptive (host or device controller), dynamic thresholding,
    correcting_x0_fn / correcting_xt_fn, denoise_to_zero, inverse(), return_intermediate, capture(), batch sharding (per
    plane: no collective; split [B, N] scales like the batch) and UniPC. A direct call of this callable returns the
    converted FDG value. Not available (ValueError before any launch and any network call): other guidance types, no
    unconditional_condition, several conditions, guidance_mask, guidance_rescale != 0, apg_eta, cfg_zero_star, cfg_pp,
    tcfg, a guidance_scale other than the default (a per-sample one included: use [B, N] fdg_scales), N outside 1..5, a
    [B, N] tensor whose B does not match x, an x the size rule refuses and DPM_Solver(reference_rounding=True).
    Not offered: diffusers' per-level parallel_weights (APG-style projection), per-level guidance rescale, a guidance
    interval."""
    assert model_type in ["noise", "x_start", "v", "score", "flow", "edm"]
    assert guidance_type in ["uncond", "classifier", "classifier-free"]
    flow_schedule = getattr(noise_schedule, "schedule", None) == "flow"
    if model_type == "flow" and not flow_schedule:
        raise ValueError("model_type='flow' needs a NoiseScheduleFlow")
    if flow_schedule and model_type in ("v", "score"):
        raise ValueError("model_type='{}' is defined for variance-preserving schedules; a NoiseScheduleFlow takes "
                         "'flow', 'noise' or 'x_start'".format(model_type))
    if flow_schedule and guidance_type == "classifier":
        raise ValueError("classifier guidance is not available with a NoiseScheduleFlow")
    edm_schedule = getattr(noise_schedule, "schedule", None) == "edm"
    if model_type == "edm" and not edm_schedule:
        raise ValueError("model_type='edm' needs a NoiseScheduleEDM")
    if edm_schedule and model_type != "edm":
        raise ValueError("a NoiseScheduleEDM takes model_type='edm' only, got '{}'".format(model_type))
    if edm_schedule and guidance_type == "classifier":
        raise ValueError("classifier guidance is not available with a NoiseScheduleEDM")
    guidance_rescale = float(guidance_rescale)
    if not math.isfinite(guidance_rescale):
        raise ValueError("guidance_rescale must be finite, got {}".format(guidance_rescale))
    if guidance_rescale != 0 and guidance_type != "classifier-free":
        raise ValueError("guidance_rescale needs guidance_type='classifier-free', got '{}'".format(guidance_type))
    apg_norm_threshold, apg_momentum = float(apg_norm_threshold), float(apg_momentum)
    if apg_eta is None:
        if apg_norm_threshold != 0 or apg_momentum != 0:
            raise ValueError("apg_norm_threshold and apg_momentum need apg_eta")
    else:
        apg_eta = float(apg_eta)
        if not (math.isfinite(apg_eta) and math.isfinite(apg_momentum)):
            raise ValueError("apg_eta and apg_momentum must be finite, got {} and {}".format(apg_eta, apg_momentum))
        if not (math.isfinite(apg_norm_threshold) and apg_norm_threshold >= 0):
            raise ValueError("apg_norm_threshold must be finite and >= 0, got {}".format(apg_norm_threshold))
    if not isinstance(cfg_zero_init_steps, int) or isinstance(cfg_zero_init_steps, bool) or cfg_zero_init_steps < 0:
        raise ValueError("cfg_zero_init_steps must be an int >= 0, got {!r}".format(cfg_zero_init_steps))
    if cfg_zero_init_steps and not cfg_zero_star:
        raise ValueError("cfg_zero_init_steps needs cfg_zero_star=True")
    for name, v in (("cfg_pp", cfg_pp), ("tcfg", tcfg), ("perp_neg", perp_neg)):
        if not isinstance(v, bool):
            raise ValueError("{} must be a bool, got {!r}".format(name, v))
    cf, many = guidance_type == "classifier-free", isinstance(condition, (list, tuple))
    options = {k for k, on in (
        ("several", cf and many and len(condition) >= 2), ("mask", guidance_mask is not None), ("perp", perp_neg),
        ("rescale", guidance_rescale != 0), ("apg", apg_eta is not None), ("cfgzero", cfg_zero_star),
        ("cfgpp", cfg_pp), ("tcfg", tcfg), ("fdg", fdg_scales is not None),
        ("per_sample", cf and _per_sample_scales(condition, guidance_scale)),
        ("zero_init", cfg_zero_init_steps > 0), ("momentum", apg_momentum != 0)) if on}
    for k in options:
        if _OPTIONS[k].needs_uc and (not cf or unconditional_condition is None):
            raise ValueError("{} needs guidance_type='classifier-free' and an unconditional_condition".format(
                _OPTIONS[k].name))
    if perp_neg and (not many or len(condition) < 2):
        raise ValueError("perp_neg needs a list of at least two conditions: the positive prompt first, then the "
                         "negatives")
    _check_options(options)
    if fdg_scales is not None:
        if torch.is_tensor(guidance_scale) or guidance_scale != 1.:
            raise ValueError("fdg_scales replaces guidance_scale, which must stay at its default 1.0, got {!r}".format(
                guidance_scale))
        _fdg_scales(fdg_scales)                       # (the form and the number of levels)
    if guidance_mask is not None:
        condition, guidance_scale, guidance_mask = _masked_arguments(condition, guidance_scale, guidance_mask)
    return WrappedModel(model, noise_schedule, model_type, model_kwargs, guidance_type, condition,
                        unconditional_condition, guidance_scale, classifier_fn, classifier_kwargs, guidance_rescale,
                        apg_eta, apg_norm_threshold, apg_momentum, cfg_zero_star, cfg_zero_init_steps, cfg_pp,
                        guidance_mask, tcfg, fdg_scales, perp_neg)


def _per_sample_scales(condition, s) -> bool:
    """Whether model_wrapper's guidance_scale holds one scale per sample: a tensor of several values for one condition,
    or a 2-D tensor or entries of several values for a list of conditions."""
    many = isinstance(condition, (list, tuple))
    if torch.is_tensor(s):
        return s.dim() >= 2 if many else s.numel() != 1
    return isinstance(s, (list, tuple)) and ((not many and len(s) != 1) or
                                             any(torch.is_tensor(v) and v.numel() != 1 for v in s))


def _masked_arguments(condition, guidance_scale, guidance_mask):
    """model_wrapper's arguments of a run with guidance masks, validated: (K conditions, their scales, K masks)."""
    many = isinstance(condition, (list, tuple))
    conds = list(condition) if many else [condition]
    masks = list(guidance_mask) if isinstance(guidance_mask, (list, tuple)) else [guidance_mask]
    if len(masks) != len(conds):
        raise ValueError("{} guidance masks for {} conditions".format(len(masks), len(conds)))
    if any(m is not None and not torch.is_tensor(m) for m in masks):
        raise ValueError("each guidance_mask entry must be a tensor or None")
    s = guidance_scale
    if not many:
        s = [float(s)] if torch.is_tensor(s) else [s]
    elif isinstance(s, (list, tuple)):
        s = [float(v) if torch.is_tensor(v) else v for v in s]
    return conds, s, masks


# =================================================================================================
# DPM_Solver
# =================================================================================================

class DPM_Solver:
    def __init__(self, model_fn, noise_schedule, algorithm_type="dpmsolver++", correcting_x0_fn=None,
                 correcting_xt_fn=None, thresholding_max_val=1., dynamic_thresholding_ratio=0.995,
                 state_dtype=None, plan_broadcast=False, predict_x0=None, thresholding=None, max_val=None,
                 reference_rounding=False):
        """Same arguments as the reference (:338-347) plus `state_dtype` and `plan_broadcast`:

        state_dtype=None keeps the reference's type promotion (fp32 state and buffers even for
        bf16/fp16 inputs, because its fp32 coefficient tensors promote every update);
        state_dtype=torch.bfloat16 / torch.float16 keeps x and the buffered model values in 16-bit
        storage (fp32 arithmetic in registers, one rounding on store) and halves HBM traffic.

        plan_broadcast=True (batch-sharded multi-GPU runs, torch.distributed initialised): rank 0
        broadcasts the scalar coefficient plan once per sample() so all ranks use bit-identical
        coefficients (distributed.py); the tensors themselves are never communicated.

        reference_rounding=True (opt-in; fp32 state, `model_type="noise"`, network returning bf16/fp16):
        reproduce the two places where the reference computes in the network's 16-bit output type -- the
        CFG combine (:329-330, three rounded ops) and, for the eps-solver, the differences of the
        buffered raw outputs (:823, :880-881, :636, :735, :741-742). Default False: both are evaluated in
        fp32 on the widened values (closer to the exact result, and the fast kernels). Runs on the
        reference-rounding instantiations of the direct vector kernels (tails and unaligned views on the
        generic kernel).

        predict_x0 / thresholding / max_val: keyword spelling of the older constructor that the JAX twin
        still uses (dpm_solver_jax.py:351): predict_x0=True selects "dpmsolver++", thresholding=True
        (valid with predict_x0) selects dynamic thresholding, max_val is `thresholding_max_val`.
        """
        if predict_x0 is not None:
            algorithm_type = "dpmsolver++" if predict_x0 else "dpmsolver"
        if thresholding:
            correcting_x0_fn = "dynamic_thresholding"
        if max_val is not None:
            thresholding_max_val = max_val
        self._wrapped = model_fn
        self.model = lambda x, t: model_fn(x, t.expand((x.shape[0])))
        self.noise_schedule = noise_schedule
        tables = getattr(noise_schedule, "log_alpha_array", None)
        if torch.is_tensor(tables) and tables.dtype != torch.float32:
            # the reference would promote x and every update to that dtype; there are no fp64 kernels
            raise TypeError("dpm_solver_b200 computes in fp32: NoiseScheduleVP(dtype={}) is not supported "
                            "by DPM_Solver".format(tables.dtype))
        assert algorithm_type in ["dpmsolver", "dpmsolver++", "sde-dpmsolver++"]
        self.algorithm_type = algorithm_type
        self._refuse(*(c for c, on in (("rr", reference_rounding), ("sde", algorithm_type == "sde-dpmsolver++"),
                                       ("eps", algorithm_type == "dpmsolver"), ("x0_fn", correcting_x0_fn is not None))
                       if on))
        if correcting_x0_fn == "dynamic_thresholding":
            self.correcting_x0_fn = self.dynamic_thresholding_fn
            self._dynamic_thresholding = True
        else:
            self.correcting_x0_fn = self._x0_hook(correcting_x0_fn)
            self._dynamic_thresholding = False
        self.correcting_xt_fn = correcting_xt_fn
        self.dynamic_thresholding_ratio = dynamic_thresholding_ratio
        self.thresholding_max_val = thresholding_max_val
        if state_dtype is not None and state_dtype not in ops.SUPPORTED_DTYPES:
            raise TypeError("state_dtype must be one of {}".format(ops.SUPPORTED_DTYPES))
        self.state_dtype = state_dtype
        self.plan_broadcast = bool(plan_broadcast)
        self.reference_rounding = bool(reference_rounding)
        if self.reference_rounding and getattr(noise_schedule, "schedule", None) in ("flow", "edm"):
            raise ValueError("reference_rounding=True reproduces the reference, which has no {} schedule".format(
                noise_schedule.schedule))
        self._rr_run = 0     # raw_round of the buffered values of the run in flight (reference_rounding)
        self._prep_cache = {}   # frozen launch descriptors of cached plan steps (ops.PreparedStep)
        self._prep_on = False

    def _options(self) -> frozenset:
        """The guidance options of the model function (none for a plain callable), and "sde" for the SDE solver."""
        w = self._wrapped
        options = w.guidance_options() if isinstance(w, WrappedModel) else frozenset()
        return options | {"sde"} if self.algorithm_type == "sde-dpmsolver++" else options

    def _refuse(self, *contexts, what=None) -> None:
        """ValueError unless the options run in the solver contexts `contexts` (_check_options)."""
        _check_options(self._options(), contexts, what)

    @staticmethod
    def _x0_hook(fn):
        """`correcting_x0_fn(x0, t)` (:379-380). The older vendored copy calls it with x0 only
        (examples/stable-diffusion/.../dpm_solver.py:447-448); a one-argument callable keeps working."""
        if fn is None or not callable(fn):
            return fn
        try:
            params = [p for p in inspect.signature(fn).parameters.values()
                      if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
            variadic = any(p.kind == p.VAR_POSITIONAL for p in inspect.signature(fn).parameters.values())
        except (TypeError, ValueError):
            return fn
        if len(params) == 1 and not variadic:
            return lambda x0, t: fn(x0)
        return fn

    def _sync_plan(self, coeffs, key=None):
        """Rank 0's coefficients on every rank. One broadcast per sampling configuration: the synced
        plan is cached under the plan key, so steady-state sample() calls issue no collective."""
        if not self.plan_broadcast:
            return coeffs
        from .distributed import broadcast_plan
        if key is None:
            return broadcast_plan(coeffs)
        cache = self.__dict__.setdefault("_synced_cache", {})
        k = (self._schedule_key(), self.algorithm_type) + key
        hit = cache.get(k)
        if hit is None:
            hit = broadcast_plan(coeffs)
            if len(cache) >= self._CACHE_MAX:
                cache.pop(next(iter(cache)))
            cache[k] = hit
        return hit

    # -- small helpers ------------------------------------------------------------------------
    @property
    def _pp(self) -> bool:
        return self.algorithm_type in ("dpmsolver++", "sde-dpmsolver++")   # data prediction

    def _sdtype(self, x) -> torch.dtype:
        if self.state_dtype is not None:
            return self.state_dtype
        if x.dtype not in ops.SUPPORTED_DTYPES:
            raise TypeError("dpm_solver_b200 supports float32, bfloat16 and float16 tensors, got {}".format(x.dtype))
        return torch.float32  # reference promotion: fp32 coefficient tensors make every update fp32

    def _state(self, x) -> torch.Tensor:
        """The tensor the kernels read as `x`. In the reference's promotion mode (state_dtype=None) a
        16-bit x is widened to fp32 for the arithmetic -- exactly what its fp32 coefficient tensors do --
        but the NETWORK still receives the caller's 16-bit tensor at that evaluation (only later states
        are fp32), so the pair is remembered for `_evaluate`."""
        sd = self._sdtype(x)
        xs = x.to(sd) if x.dtype != sd else x
        xs = xs if ops.CudaBackend._layout(xs) is not None else xs.contiguous()
        # (re-evaluations at the same state -- a rejected adaptive step -- must see it again: the pair stays
        # until the next _state() call or the end of sample())
        if self.state_dtype is None and x.dtype != sd:
            self._net_input = (xs, x)
        elif self.__dict__.get("_net_input") is not None and self._net_input[0] is not xs:
            self._net_input = None
        return xs

    def _alpha_sigma(self, t_host):
        ns = self.noise_schedule
        return float(ns.marginal_alpha(t_host)), float(ns.marginal_std(t_host))

    # -- model evaluation ---------------------------------------------------------------------
    def _evaluate(self, x, t_dev, t_input=None) -> RawOutput:
        """Call the user's network at (x, t); same call the reference makes through self.model. CFG-Zero*'s zero-init
        evaluations of a run return a raw output of 0 instead, without calling it."""
        w = self._wrapped
        if self.__dict__.get("_cfz_left"):
            self._cfz_left -= 1
            return RawOutput(self._cfz_zeros(x), None, PARAM_BY_NAME[w.model_type], 1.0)
        orig = self.__dict__.get("_net_input")
        if orig is not None and orig[0] is x:
            x = orig[1]                           # the caller's own (16-bit) tensor, as the reference passes it
        if isinstance(w, WrappedModel) and w.fusable:
            pair = self.__dict__.get("_xin_pair")
            x_in = pair[1] if (pair is not None and pair[0] is x) else None
            # (the continuous label is only read when no precomputed model-input time row is handed over)
            return w.raw(x, t_dev.expand((x.shape[0])) if t_input is None else None, t_input, x_in)
        return RawOutput(self.model(x, t_dev), None, PARAM_NOISE, 1.0)

    def _dup_target(self, x):
        """Under CFG the network consumes cat([x]*2) (:326), cat([x]*(K+1)) with K >= 2 conditions. When nothing can
        touch x between the update and the next evaluation, the update kernel writes x_t straight into every block of
        a [copies*B, ...] buffer: returns (x_in, block 0, block 1, ...) or None."""
        w = self._wrapped
        if self.correcting_xt_fn is not None or not (isinstance(w, WrappedModel) and w.fusable and w.uses_cfg):
            return None
        B, n = x.shape[0], 2 if w.cond_scales is None else len(w.cond_scales) + 1
        shape = (n * B,) + tuple(x.shape[1:])
        if ops.CudaBackend._layout(x) == "cl":      # keep a channels_last network's layout
            x_in = torch.empty(shape, dtype=x.dtype, device=x.device,
                               memory_format=torch.channels_last if x.dim() == 4 else torch.channels_last_3d)
        else:
            x_in = torch.empty(shape, dtype=x.dtype, device=x.device)
        if n == 2:
            return x_in, x_in[:B], x_in[B:]
        return (x_in,) + tuple(x_in[i * B:(i + 1) * B] for i in range(n))

    _CACHE_MAX = 16

    def _schedule_key(self):
        """Identity of the schedule the cached plans were computed from. The table tensors are pinned
        in `_schedule_refs` so their ids cannot be recycled; `_version` catches in-place edits."""
        ns = self.noise_schedule
        if getattr(ns, "schedule", None) == "discrete":
            la, ta = ns.log_alpha_array, ns.t_array
            refs = self.__dict__.setdefault("_schedule_refs", {})
            refs[id(la)], refs[id(ta)] = la, ta
            if len(refs) > 64:
                for k in list(refs)[:-8]:
                    refs.pop(k)
                for name in ("_plan_cache", "_table_cache", "_synced_cache"):
                    self.__dict__.pop(name, None)
            return ("discrete", id(la), la._version, id(ta), ta._version, ns.total_N)
        return (getattr(ns, "schedule", None), getattr(ns, "beta_0", None), getattr(ns, "beta_1", None),
                getattr(ns, "T", None), getattr(ns, "shift", None), getattr(ns, "time_scale", None)) + \
            tuple(getattr(ns, k, None) for k in ("sigma_min", "sigma_max", "sigma_data", "rho", "total_N"))

    def _plan_id(self, key):
        """Hashable identity of a cached plan (schedule + algorithm + sampling arguments): prepared launches are
        keyed by it, so a changed schedule or argument never meets a stale descriptor."""
        return (self._schedule_key(), self.algorithm_type, self.plan_broadcast) + key

    def _host_plan(self, key, build):
        """Coefficient plan of a run, cached per (schedule, algorithm, sampling arguments): repeated
        sample() calls with the same configuration (serving) skip the host scalar work entirely."""
        cache = self.__dict__.setdefault("_plan_cache", {})
        k = (self._schedule_key(), self.algorithm_type) + key
        hit = cache.get(k)
        if hit is None:
            hit = build()
            if len(cache) >= self._CACHE_MAX:
                cache.pop(next(iter(cache)))
            cache[k] = hit
        return hit

    def _device_tables(self, key, t_host, batch, device, n_eval=None):
        """Device copies of the time grid and of the model-input time matrix, cached with the plan
        (they depend on the batch size, the network's input rows and the device only)."""
        cache = self.__dict__.setdefault("_table_cache", {})
        k = (self._schedule_key(), self.algorithm_type) + key + (batch, self._input_rows(batch), str(device),
                                                                 id(self._wrapped))
        hit = cache.get(k)
        if hit is None:
            t_dev = self._upload(t_host, device)
            tin = self._input_times(t_host if n_eval is None else t_host[:n_eval], batch, device)
            # the per-step views are built once here: indexing a device tensor costs ~1.5 us of host time, three
            # times per solver step
            n = t_dev.shape[0]
            hit = (t_dev, tin, [t_dev[i] for i in range(n)], [t_dev[i:i + 1] for i in range(n)],
                   None if tin is None else [tin[i] for i in range(tin.shape[0])])
            if len(cache) >= self._CACHE_MAX:
                cache.pop(next(iter(cache)))
            cache[k] = hit
        return hit

    def _denoise_tables(self, t_0, batch, device):
        """(device label (1,), model-input time row or None, (alpha, sigma)) of the denoise-to-zero tail."""
        cache = self.__dict__.setdefault("_table_cache", {})
        k = (self._schedule_key(), "d2z", float(t_0), batch, self._input_rows(batch), str(device), id(self._wrapped))
        hit = cache.get(k)
        if hit is None:
            th = torch.ones((1,)) * t_0                                   # fp32, as `torch.ones((1,)).to(device) * t_0`
            tin = self._input_times(th, batch, device)
            hit = (self._upload(th, device), None if tin is None else tin[0], self._alpha_sigma(th))
            if len(cache) >= self._CACHE_MAX:
                cache.pop(next(iter(cache)))
            cache[k] = hit
        return hit

    def _input_rows(self, batch: int) -> int:
        """Rows of the network input for a batch: 2B under CFG, B when a one-element scale tensor now holds 1 and the
        halves are bypassed. It can change between runs of one solver (the tensor edited in place, or the wrapper's
        settings changed), so the model-input time tables are keyed by it."""
        w = self._wrapped
        return w.input_rows(batch) if isinstance(w, WrappedModel) and w.fusable else batch

    @staticmethod
    def _upload(t_host: torch.Tensor, device):
        """Host vector -> device without draining the stream (pinned staging, async copy)."""
        device = torch.device(device)
        if device.type != "cuda":
            return t_host.to(device)
        return t_host.pin_memory().to(device, non_blocking=True)

    def _input_times(self, t_host: torch.Tensor, batch: int, device):
        """[n_evals, rows] device matrix of model-input times for a whole run (one tiny kernel per
        sample() instead of two per model call); None when the model takes t_continuous itself."""
        w = self._wrapped
        if not (isinstance(w, WrappedModel) and w.fusable and w.noise_schedule.schedule in ('discrete', 'flow', 'edm')):
            return None
        t_in = self._upload(w.get_model_input_time(t_host.reshape(-1)), device)   # (t - 1/N) * 1000, fp32, :278
        return t_in[:, None].expand(t_in.shape[0], w.input_rows(batch)).contiguous()

    def _conv_args(self, raw: RawOutput, xe, alsig, sdtype, x0: bool) -> StepArgs:
        """StepArgs fields that turn `raw` into the buffered model value at time t (x0 if `x0`, else
        eps). `alsig` is (alpha_t, sigma_t) from the plan, or the host time tensor to derive them."""
        if raw.is_x0:
            # identity on the materialised x0, for every value: x0 = (-0) - (-1)*e_cond (then the clamp)
            return StepArgs(n_model=1, e_cond=raw.e_cond, param=PARAM_FLOW, predict_x0=True, alpha_e=1.0, sigma_e=-1.0,
                            xe=torch.full_like(xe, -0.0), state_dtype=sdtype)
        a = StepArgs(n_model=2 if raw.e_uncond is not None else 1, e_cond=raw.e_cond,
                     e_uncond=raw.e_uncond, param=raw.param, guidance=raw.guidance,
                     predict_x0=x0, state_dtype=sdtype)
        if x0 or raw.param != PARAM_NOISE:
            if alsig is _DEV:
                pass        # (alpha_t, sigma_t) arrive with the launch's device coefficient block (StepArgs.coef_dev)
            else:
                a.alpha_e, a.sigma_e = alsig if isinstance(alsig, tuple) else self._alpha_sigma(alsig)
                if raw.param == PARAM_EDM:
                    a.alpha_e, a.sigma_e = self._wrapped.noise_schedule.conversion_words(a.alpha_e, a.sigma_e, x0)
            a.xe = xe
        return a

    @staticmethod
    def _needs_conversion(raw: RawOutput, sdtype, x0: bool) -> bool:
        return x0 or raw.e_uncond is not None or raw.param != PARAM_NOISE or raw.e_cond.dtype != sdtype

    _RR_CODE = {torch.bfloat16: 1, torch.float16: 2}      # dpm_dtype codes carried by raw_round

    def _rr_code(self, raw: RawOutput) -> int:
        """16-bit dtype code of raw NOISE outputs in reference-rounding mode, else 0."""
        if not self.reference_rounding or self.state_dtype is not None or raw.param != PARAM_NOISE:
            return 0
        return self._RR_CODE.get(raw.e_cond.dtype, 0)

    @staticmethod
    def _rr_coeffs(co: P.Coeffs, code: int) -> P.Coeffs:
        """singlestep-3 'taylor' (:780-783) in reference-rounding mode: r1, r2 that arrive as 0-dim tensors
        (the sample() loop, :1223-1227) are cast to the buffers' 16-bit type where they are the LEFT operand
        of a product (`(1./r1) * (..)`, `r2 * D1_0`, `r1 * D1_1`); python floats (the defaults of the
        directly called method) and right-hand scalars (the divisor `r2 - r1`) enter in fp32 -- torch's CPU
        kernels keep the second operand of mul/div in the op's fp32 math type when it is a scalar."""
        if co.form != FORM_SS3T or not co.r_tensor:
            return co
        T = torch.bfloat16 if code == 1 else torch.float16
        rT = lambda v: float(torch.tensor(v, dtype=torch.float32).to(T))
        r1t, r2t = bool(co.r_tensor & 1), bool(co.r_tensor & 2)
        return dataclasses.replace(co, w0=rT(co.w0) if r1t else co.w0, w1=rT(co.w1) if r2t else co.w1,
                                   w2=rT(co.w2) if r2t else co.w2, w3=rT(co.w3) if r1t else co.w3,
                                   w4=co.w4)

    def _post_model(self, raw: RawOutput, xe, t_dev, alsig, co: Optional[P.Coeffs] = None, x=None,
                    m1=None, m2=None, want_m: bool = True, dup_out: bool = False, x0: Optional[bool] = None,
                    slot=None):
        """The fused post-model step: buffered value from `raw` (+ optional update `co`).

        Returns (m_new, x_next). Falls back to two launches only when a user-supplied
        `correcting_x0_fn` must see the materialised x0 (:440-441).

        `slot` names a step of a CACHED coefficient plan (sample() loops): its launch descriptor is frozen after
        the first run (ops.PreparedStep) and later runs only patch tensor pointers -- the steady-state host path."""
        be = ops.backend()
        guided = (raw.form, raw.consts)
        if raw.form == "fdg":
            # frequency-decoupled guidance: the pyramid pass over both raw halves (+1 launch) gives g in the network's
            # dtype, handed on as one network output of the same parameterisation; everything below is the one-output
            # path (the fused step with out / out2, the quantile, UniPC, device coefficients)
            raw = _fdg_output(be, raw)
        if raw.form == "perp":
            # Perp-Neg: the words pass over the K+1 raw outputs (+2 launches) gives condition 1's per-sample weight;
            # from here on the evaluation is a regional-guidance one (the masked fused step with its replicas, the fp32
            # materialisation for the quantile, the correcting_x0_fn split, device coefficients)
            raw = _perp_output(be, raw)
        pkey = None
        if slot is not None and self._prep_on:
            # (the guidance form and its constants are part of the key: a launch frozen for one form never serves
            # another)
            # (and so is a per-sample scale: a guided evaluation never meets a launch frozen with one scale)
            # (and so are the scales of several conditions: such a step is never frozen, and a key with them cannot
            # meet a launch frozen for one condition)
            # (and so is dynamic thresholding: a launch frozen without the clamp never serves a solver switched to it)
            pkey = (slot, raw.param, raw.guidance, raw.scales, raw.guidance_b is None, raw.e_uncond is None,
                    raw.e_cond.dtype, xe.dtype, xe.shape, want_m, dup_out, self._dynamic_thresholding, guided)
            prep = self._prep_cache.get(pkey)
            if prep is not None:
                r = prep.launch((x, xe, raw.e_cond, m1, m2, raw.e_cond, raw.e_uncond))
                if r is not None:
                    m_new, x_next, x_in = r
                    if x_in is not None:
                        self._xin_pair = (x_next, x_in)
                    if m_new is None and prep.d.n_model == 0:
                        m_new = raw.e_cond                  # pure update on the raw noise: it IS the buffered value
                    return m_new, x_next
        if raw.form == "cfgpp" and co is not None:
            return self._cfgpp_step(raw, xe, alsig, co, x, m1, want_m, dup_out)
        x0 = self._pp if x0 is None else x0          # buffered value: x0 (dpmsolver++ / data_prediction_fn) or eps
        sd = xe.dtype if xe is not None else (x.dtype if x is not None else raw.e_cond.dtype)
        custom_fix = x0 and self.correcting_x0_fn is not None and not self._dynamic_thresholding
        thresholded = x0 and self._dynamic_thresholding
        code = self._rr_code(raw)
        rr = 0
        q_raw = None        # what the quantile reads, when not `raw` itself
        apg_a = None        # the step arguments of an adaptive-projected-guidance evaluation
        split = False       # the buffered value and the update in two launches
        if raw.form == "apg":
            # the words pass (+2 launches), then the fused step. With dynamic thresholding (the quantile takes one
            # plain combine) the guided x0 is materialised once in fp32 (+1 launch) and handed on as one network output.
            # Under UniPC, whose launch converts at its own state and takes one network output, a FORM_NONE launch
            # writes the buffered value and the UniPC launch reads it as a pure update.
            if alsig is _DEV:
                if co is None or co.dev is None:
                    raise RuntimeError("device-side scalars need the coefficient block of the consuming launch")
                marg, cdev = None, co.dev
            else:
                marg, cdev = (alsig if isinstance(alsig, tuple) else self._alpha_sigma(alsig)), None
            r_prev, r_out = self._apg_buffers(raw, xe)
            xa = xe.float() if thresholded and xe.dtype != torch.float32 else xe
            a = _apg_args(be, raw, xa, marg, torch.float32 if thresholded else sd, x0, self._wrapped.noise_schedule,
                          cdev, r_prev, r_out)
            if thresholded:
                a.form = FORM_NONE
                raw = RawOutput(be.step(a)[0], None, PARAM_NOISE, 1.0, is_x0=x0)
                split = self._apg_materialise
            elif self._apg_materialise:
                a.form = FORM_NONE
                m_new = be.step(a)[0]
                if custom_fix:
                    m_new = self._state_like(self.correcting_x0_fn(m_new, t_dev), sd)
                if co is None:
                    return m_new, None
                b = StepArgs(n_model=0, m0=m_new, state_dtype=sd)
                self._fill_update(b, co, x, m1, m2)
                dup = self._dup_target(x) if dup_out else None
                if dup is not None:
                    b.out, b.out2 = dup[1], dup[2]
                x_next = be.step(b)[1]
                if dup is not None:
                    self._xin_pair = (x_next, dup[0])
                return m_new, x_next
            else:
                apg_a = a
        words = _words(be, raw)     # guidance rescale, CFG-Zero*, TCFG: the per-sample words pass (+2 launches)
        if code:
            # reference-rounding mode (raw 16-bit NOISE outputs, fp32 state): bits 0-1 make the fused kernel take the
            # CFG combine in the network's type, three rounded ops (:329-330); for the eps-solver the buffered values
            # are those raw outputs, so bit 2 makes their differences round too (:823, :880-881, :636, :735)
            rr = code
            if not x0:
                rr = self._rr_run = code | 4
        if raw.e_uncond is not None and (thresholded or (self._apg_materialise and raw.form in ("cfgzero", "tcfg"))):
            # one fp32 output for the quantile kernels, which take the plain fp32 combine with one scale, and for UniPC,
            # whose launch takes one network output and converts at its own state (+1 launch)
            if words is not None or code:
                # the reference's rounded noise, or the rescaled, CFG-Zero* or TCFG combine of the raw outputs, then
                # treated as one network output (the parameterisation, which the quantile and the step apply, still
                # converts it)
                a = StepArgs(form=FORM_NONE, n_model=2, e_cond=raw.e_cond, e_uncond=raw.e_uncond, param=PARAM_NOISE,
                             guidance=raw.guidance, state_dtype=torch.float32, raw_round=code)
                raw = RawOutput(be.step(_guidance_args(a, words, raw))[0], None, raw.param, 1.0)
                words, rr = None, 0
            elif raw.guidance_b is not None or raw.e_conds is not None:
                # per-sample scales: the guided noise, each half parameterised, then combined with its sample's scale,
                # as the reference orders it; several conditions: their combined noise, each block parameterised first.
                # (a flow or EDM network's outputs are converted to x0 directly and combined as x0: no eps -> x0
                # follows)
                flow = raw.param in (PARAM_FLOW, PARAM_EDM)
                a = self._conv_args(raw, xe, alsig, torch.float32, flow)
                if a.xe is not None and a.xe.dtype != torch.float32:
                    a.xe = a.xe.float()
                if alsig is _DEV:
                    if co is None or co.dev is None:
                        raise RuntimeError("device-side scalars need the coefficient block of the consuming launch")
                    a.coef_dev = co.dev
                e = be.step(_guidance_args(a, None, raw))[0]
                if raw.e_conds is not None:
                    # several conditions: the quantile reads the materialised noise; the step then recomputes the same
                    # fp32 combine from the K+1 outputs, so that it can also write the K+1 blocks of the next input
                    q_raw = RawOutput(e, None, PARAM_NOISE, 1.0, is_x0=flow)
                else:
                    raw = RawOutput(e, None, PARAM_NOISE, 1.0, is_x0=flow)
        if (rr & 4) and co is not None:
            co = self._rr_coeffs(co, code)
        if not self._needs_conversion(raw, sd, x0):
            m_new = raw.e_cond if ops.CudaBackend._layout(raw.e_cond) is not None else raw.e_cond.contiguous()
            x_next = self._pure_update(co, x, m_new, m1, m2, rr=rr & 4 and rr, pkey=pkey if m_new is raw.e_cond else None) \
                if co is not None else None
            return m_new, x_next
        a = apg_a if apg_a is not None else _guidance_args(self._conv_args(raw, xe, alsig, sd, x0), words, raw)
        if alsig is _DEV:
            if co is None or co.dev is None:
                raise RuntimeError("device-side scalars need the coefficient block of the consuming launch")
            a.coef_dev = co.dev
        if x0 and self._dynamic_thresholding:
            a.per_sample = xe.numel() // xe.shape[0]
            qa = a
            if q_raw is not None:
                qa = self._conv_args(q_raw, xe, alsig, sd, x0)
                qa.per_sample, qa.coef_dev = a.per_sample, a.coef_dev
            a.thr = be.dynamic_threshold(qa, float(self.dynamic_thresholding_ratio),
                                         float(self.thresholding_max_val))
        if custom_fix or co is None or split:
            a.form = FORM_NONE
            a.raw_round = rr & 3
            m_new = be.step(a)[0]
            if custom_fix:
                m_new = self._state_like(self.correcting_x0_fn(m_new, t_dev), sd)
            x_next = self._pure_update(co, x, m_new, m1, m2, rr=rr & 4 and rr) if co is not None else None
            return m_new, x_next
        self._fill_update(a, co, x, m1, m2)
        a.sde = self.__dict__.get("_sde_noise")
        a.want_m_out = want_m
        a.raw_round = rr
        dup = self._dup_target(x) if dup_out else None
        if dup is not None:
            if a.e_conds is not None:
                a.out, a.replicas = dup[1], dup[2:]     # blocks 1..K of the next network input
            else:
                a.out, a.out2 = dup[1], dup[2]
        m_new, x_next = be.step(a)
        if dup is not None:
            self._xin_pair = (x_next, dup[0])
        if pkey is not None and not a.per_sample and a.e_conds is None:
            self._remember(pkey, a, dup)
        return m_new, x_next

    _apg_materialise = False     # UniPC: its launch takes one network output, so an APG or CFG-Zero* value is
                                 # materialised first

    def _check_fdg(self, x) -> None:
        """Frequency-decoupled guidance: x's shape against the size rule and the per-sample rows, before any launch."""
        w = self._wrapped
        if isinstance(w, WrappedModel) and w.fdg_levels:
            w.fdg_args(x)

    def _cfgpp_step(self, raw: RawOutput, xe, alsig, co: P.Coeffs, x, m1, want_m: bool, dup_out: bool):
        """A CFG++ update (dpm_step_cfgpp, one launch): returns (U, x_next), U the x0 of the unconditional output alone,
        which the multistep loop buffers in place of the guided x0."""
        if co.form not in (FORM_LIN1, ops.FORM_DIFF2) or co.c0_on_old or co.dev is not None:
            raise ValueError("cfg_pp takes DPM-Solver++ multistep updates of order 1 or 2")
        a = _guidance_args(self._conv_args(raw, xe, alsig, xe.dtype, True), None, raw)
        self._fill_update(a, co, x, m1, None)
        a.cfgpp_g, a.want_m_out = co.g, want_m
        dup = self._dup_target(x) if dup_out else None
        if dup is not None:
            a.out, a.out2 = dup[1], dup[2]
        m_new, x_next = ops.backend().step(a)
        if dup is not None:
            self._xin_pair = (x_next, dup[0])
        return m_new, x_next

    def _apg_buffers(self, raw: RawOutput, xe):
        """(r_prev, r_out) of an APG evaluation. Without momentum, or outside a sample() / inverse() run: (None, None).
        The first evaluation of a run allocates the run's fp32 buffer and writes it without reading it (so a captured
        graph needs no reset launch); later ones update it in place."""
        if raw.consts[2] == 0 or not self.__dict__.get("_apg_run"):
            return None, None
        r = self.__dict__.get("_apg_r")
        if r is None:
            self._apg_r = torch.empty_like(xe, dtype=torch.float32)
            return None, self._apg_r
        return r, r

    @contextlib.contextmanager
    def _apg_scope(self):
        """One sample() / inverse() run: the APG momentum buffer lives for its duration, and so do CFG-Zero*'s count of
        zero-init evaluations left and its zero outputs."""
        self._apg_run, self._apg_r = True, None
        self._cfz_left = self._wrapped.cfg_zero_init_steps if "zero_init" in self._options() else 0
        self._cfz_zero = {}
        try:
            yield
        finally:
            self._apg_run, self._apg_r = False, None
            self._cfz_left, self._cfz_zero = 0, {}

    def _cfz_zeros(self, x):
        """The raw output 0 of a zero-init evaluation at state x: laid out like x, allocated once per run and
        (shape, dtype, layout), and only ever read."""
        key = (tuple(x.shape), x.dtype, x.stride(), x.device)
        z = self._cfz_zero.get(key)
        if z is None:
            z = self._cfz_zero[key] = torch.zeros_like(x)
        return z

    def _remember(self, pkey, a: StepArgs, dup=None) -> None:
        """Freeze the launch that just ran as the prepared form of its plan step."""
        if dup is not None:
            a.out, a.out2 = dup[1], dup[2]
        prep = ops.backend().prepare(a)
        if prep is not None:
            if len(self._prep_cache) >= 512:
                self._prep_cache.clear()
            self._prep_cache[pkey] = prep

    @staticmethod
    def _state_like(t, sd):
        if t.dtype != sd:
            t = t.to(sd)
        return t if ops.CudaBackend._layout(t) is not None else t.contiguous()   # dense (row-major / channels_last)

    @staticmethod
    def _fill_update(a: StepArgs, co: P.Coeffs, x, m1, m2) -> None:
        a.form, a.x, a.m1, a.m2 = co.form, x, m1, m2
        if co.dev is not None:
            a.coef_dev = co.dev
        a.a, a.c0, a.c1, a.c2 = co.a, co.c0, co.c1, co.c2
        a.w0, a.w1, a.w2, a.w3, a.w4 = co.w0, co.w1, co.w2, co.w3, co.w4
        a.c0_on_old = co.c0_on_old

    def _pure_update(self, co: P.Coeffs, x, m0, m1=None, m2=None, rr: Optional[int] = None, pkey=None):
        if rr is None:
            # directly called update methods: buffers handed over in one 16-bit type are raw outputs
            rr = 0
            dts = {m.dtype for m in (m0, m1, m2) if m is not None}
            if (self.reference_rounding and self.state_dtype is None and x.dtype == torch.float32
                    and len(dts) == 1 and next(iter(dts)) in self._RR_CODE):
                rr = self._RR_CODE[next(iter(dts))] | 4
        a = StepArgs(n_model=0, m0=self._state_like(m0, x.dtype), state_dtype=x.dtype, raw_round=rr)
        self._fill_update(a, co, x, None if m1 is None else self._state_like(m1, x.dtype),
                          None if m2 is None else self._state_like(m2, x.dtype))
        a.sde = self.__dict__.get("_sde_noise")
        out = ops.backend().step(a)[1]
        if pkey is not None and not rr:
            self._remember(pkey, a)
        return out

    # -- reference API: model functions ---------------------------------------------------------
    def dynamic_thresholding_fn(self, x0, t):
        """Imagen dynamic thresholding of a materialised x0 (:416-425)."""
        x0c = self._state_like(x0, x0.dtype if x0.dtype in ops.SUPPORTED_DTYPES else torch.float32)
        # x0 = (x0 - 0*0)/1 exactly: reuse the conversion path with eps = 0
        zeros = torch.zeros_like(x0c)
        a = StepArgs(form=FORM_NONE, n_model=1, e_cond=zeros, xe=x0c, predict_x0=True, alpha_e=1.0,
                     sigma_e=0.0, state_dtype=x0c.dtype, per_sample=x0c.numel() // x0c.shape[0])
        be = ops.backend()
        a.thr = be.dynamic_threshold(a, float(self.dynamic_thresholding_ratio), float(self.thresholding_max_val))
        return be.step(a)[0]

    def noise_prediction_fn(self, x, t):
        """Return the noise prediction model (:427-431)."""
        if self.reference_rounding:
            # the conversion launch, so that a 16-bit CFG combine is rounded as the reference rounds it (:329-330)
            xs = self._state(x)
            return self._post_model(self._evaluate(xs, t), xs, t, P._cpu(t)[:1], x0=False)[0]
        return self.model(x, t)

    def data_prediction_fn(self, x, t):
        """x0 = (x - sigma_t*eps)/alpha_t with corrector (:433-442), one fused launch."""
        xs = self._state(x)
        raw = self._evaluate(xs, t)
        return self._post_model(raw, xs, t, P._cpu(t)[:1], x0=True)[0]   # x0 regardless of algorithm_type

    def model_fn(self, x, t):
        """Noise prediction (dpmsolver) or data prediction (dpmsolver++) (:444-451)."""
        if self._pp:
            return self.data_prediction_fn(x, t)
        xs = self._state(x)
        raw = self._evaluate(xs, t)
        return self._post_model(raw, xs, t, P._cpu(t)[:1])[0]

    # -- reference API: time grids ---------------------------------------------------------------
    def get_time_steps(self, skip_type, t_T, t_0, N, device):
        """Time grid of N+1 points (:453-480). Computed on the host, moved to `device`.

        skip_type='karras' (not in the reference; every schedule): Karras et al.'s rho = 7 spacing of the noise level
        s = exp(-lambda) (the VE sigma, sigma_t/alpha_t): with lambda_T, lambda_0 taken as 'logSNR' takes them,
        r = linspace(exp(-lambda_T/7), exp(-lambda_0/7), N+1)^7 in fp32 (ends formed in double) and the grid is
        inverse_lambda(-log(r)), with no endpoint pinning, like 'logSNR'. This is the "Karras" spacing of DPM-Solver++
        front ends; on a discrete VP schedule the labels are not rounded to integer timesteps (diffusers rounds them),
        so the grid differs from diffusers' there."""
        if skip_type == 'karras':
            lambda_T = self.noise_schedule.marginal_lambda(torch.tensor(t_T)).item()
            lambda_0 = self.noise_schedule.marginal_lambda(torch.tensor(t_0)).item()
            r = torch.linspace(math.exp(-lambda_T / 7.), math.exp(-lambda_0 / 7.), N + 1).pow(7.)
            return self.noise_schedule.inverse_lambda(-torch.log(r)).to(device)
        if skip_type == 'logSNR':
            lambda_T = self.noise_schedule.marginal_lambda(torch.tensor(t_T))
            lambda_0 = self.noise_schedule.marginal_lambda(torch.tensor(t_0))
            logSNR_steps = torch.linspace(lambda_T.item(), lambda_0.item(), N + 1)
            return self.noise_schedule.inverse_lambda(logSNR_steps).to(device)
        elif skip_type == 'time_uniform':
            return torch.linspace(t_T, t_0, N + 1).to(device)
        elif skip_type == 'time_quadratic':
            t_order = 2
            return torch.linspace(t_T ** (1. / t_order), t_0 ** (1. / t_order), N + 1).pow(t_order).to(device)
        else:
            raise ValueError("Unsupported skip_type {}, need to be 'logSNR' or 'time_uniform' or "
                             "'time_quadratic' or 'karras'".format(skip_type))

    def get_orders_and_timesteps_for_singlestep_solver(self, steps, order, skip_type, t_T, t_0, device):
        """Orders and outer grid of 'DPM-Solver-fast' (:482-539)."""
        orders = P.singlestep_orders(steps, order)
        if skip_type == 'logSNR':
            timesteps_outer = self.get_time_steps(skip_type, t_T, t_0, len(orders), device)
        else:
            idx = torch.cumsum(torch.tensor([0, ] + orders), 0).to(device)
            timesteps_outer = self.get_time_steps(skip_type, t_T, t_0, steps, device)[idx]
        return timesteps_outer, orders

    def denoise_to_zero_fn(self, x, s):
        """Final first-order denoise to t=0 (:541-545)."""
        return self.data_prediction_fn(x, s)

    # -- reference API: single updates (direct-call path; scalars computed per call) -------------
    def dpm_solver_first_update(self, x, s, t, model_s=None, return_intermediate=False):
        """DPM-Solver-1 / DDIM step s -> t (:547-592)."""
        self._refuse("direct", what="dpm_solver_first_update()")
        x = self._state(x)
        co = P.first_update_coeffs(self.noise_schedule, self.algorithm_type, s, t)
        if model_s is None:
            raw = self._evaluate(x, s)
            model_s, x_t = self._post_model(raw, x, s, P._cpu(s), co, x, want_m=return_intermediate)
        else:
            x_t = self._pure_update(co, x, model_s)
        if return_intermediate:
            return x_t, {'model_s': model_s}
        return x_t

    def _device_time(self, t_host, like):
        return t_host.to(like.device)

    def singlestep_dpm_solver_second_update(self, x, s, t, r1=0.5, model_s=None, return_intermediate=False,
                                            solver_type='dpmsolver'):
        """Singlestep DPM-Solver-2 s -> t (:594-673)."""
        self._refuse("direct", what="singlestep_dpm_solver_second_update()")
        if solver_type not in ['dpmsolver', 'taylor']:
            raise ValueError("'solver_type' must be either 'dpmsolver' or 'taylor', got {}".format(solver_type))
        sp = P.singlestep_second(self.noise_schedule, self.algorithm_type, solver_type, s, t, r1)
        x_t, ms = self._run_singlestep(self._state(x), sp, model_s=model_s, keep=return_intermediate)
        if return_intermediate:
            return x_t, {'model_s': ms[0], 'model_s1': ms[1]}
        return x_t

    def singlestep_dpm_solver_third_update(self, x, s, t, r1=1. / 3., r2=2. / 3., model_s=None, model_s1=None,
                                           return_intermediate=False, solver_type='dpmsolver'):
        """Singlestep DPM-Solver-3 s -> t (:675-794)."""
        self._refuse("direct", what="singlestep_dpm_solver_third_update()")
        if solver_type not in ['dpmsolver', 'taylor']:
            raise ValueError("'solver_type' must be either 'dpmsolver' or 'taylor', got {}".format(solver_type))
        sp = P.singlestep_third(self.noise_schedule, self.algorithm_type, solver_type, s, t, r1, r2)
        x_t, ms = self._run_singlestep(self._state(x), sp, model_s=model_s, model_s1=model_s1,
                                       keep=return_intermediate)
        if return_intermediate:
            return x_t, {'model_s': ms[0], 'model_s1': ms[1], 'model_s2': ms[2]}
        return x_t

    def _run_singlestep(self, x, sp: P.SinglestepPlan, model_s=None, model_s1=None, keep=False,
                        times_dev: Optional[List[torch.Tensor]] = None, alsig=None, t_inputs=None,
                        dup_last: bool = False, slot=None):
        """Execute one singlestep update: one fused launch per model evaluation.

        Stage j converts the network output evaluated at (x_j, times[j]) and, in the same kernel,
        produces the next intermediate state from the base state x (:630-640, :723-750)."""
        td = times_dev if times_dev is not None else [self._device_time(tt, x) for tt in sp.times]
        als = alsig if alsig is not None else sp.times
        tin = t_inputs if t_inputs is not None else [None] * len(sp.times)
        ms: List[Optional[torch.Tensor]] = [model_s, model_s1, None]
        taylor3 = sp.order == 3 and sp.stages[-1].form == FORM_SS3T
        xe = x
        x_next = None
        for j, co in enumerate(sp.stages):
            last = j == len(sp.stages) - 1
            # buffers the stage reads besides the value it computes itself
            if co.form == FORM_LIN1:
                m1 = m2 = None
            elif co.form == FORM_SS3T:
                m1, m2 = ms[1], ms[0]
            else:
                m1, m2 = ms[0], None
            given = ms[j] if j < 2 else None
            # x_s1 is not needed when the caller already supplies model_s1 (:722)
            skip_update = j == 0 and sp.order == 3 and ms[1] is not None
            if given is not None:
                # caller supplied this model value (the adaptive solver reuses the lower-order ones)
                if not skip_update:
                    x_next = self._pure_update(co, x, given, m1, m2, rr=self._rr_run)
            else:
                raw = self._evaluate(xe, td[j], tin[j])
                want = keep or (not last and (j == 0 or taylor3))
                if skip_update:
                    m_new, _ = self._post_model(raw, xe, td[j], als[j])
                else:
                    m_new, x_next = self._post_model(raw, xe, td[j], als[j], co, x, m1, m2, want_m=want,
                                                     dup_out=(not last) or dup_last,
                                                     slot=None if slot is None else slot + (j,))
                ms[j] = m_new
            xe = x_next
        return x_next, ms

    def multistep_dpm_solver_second_update(self, x, model_prev_list, t_prev_list, t, solver_type="dpmsolver"):
        """Multistep DPM-Solver-2 (:796-852)."""
        self._refuse("direct", what="multistep_dpm_solver_second_update()")
        if solver_type not in ['dpmsolver', 'taylor']:
            raise ValueError("'solver_type' must be either 'dpmsolver' or 'taylor', got {}".format(solver_type))
        co = P.multistep_coeffs(self.noise_schedule, self.algorithm_type, solver_type, 2, t_prev_list, t)
        return self._pure_update(co, self._state(x), model_prev_list[-1], model_prev_list[-2])

    def multistep_dpm_solver_third_update(self, x, model_prev_list, t_prev_list, t, solver_type='dpmsolver'):
        """Multistep DPM-Solver-3 (:854-904); needs exactly three buffered values."""
        self._refuse("direct", what="multistep_dpm_solver_third_update()")
        model_prev_2, model_prev_1, model_prev_0 = model_prev_list
        t_prev_2, t_prev_1, t_prev_0 = t_prev_list
        co = P.multistep_coeffs(self.noise_schedule, self.algorithm_type, solver_type, 3,
                                [t_prev_2, t_prev_1, t_prev_0], t)
        return self._pure_update(co, self._state(x), model_prev_0, model_prev_1, model_prev_2)

    def singlestep_dpm_solver_update(self, x, s, t, order, return_intermediate=False, solver_type='dpmsolver',
                                     r1=None, r2=None):
        """Order dispatch (:906-930)."""
        self._refuse("direct", what="singlestep_dpm_solver_update()")
        if order == 1:
            return self.dpm_solver_first_update(x, s, t, return_intermediate=return_intermediate)
        elif order == 2:
            return self.singlestep_dpm_solver_second_update(x, s, t, return_intermediate=return_intermediate,
                                                            solver_type=solver_type, r1=r1)
        elif order == 3:
            return self.singlestep_dpm_solver_third_update(x, s, t, return_intermediate=return_intermediate,
                                                           solver_type=solver_type, r1=r1, r2=r2)
        else:
            raise ValueError("Solver order must be 1 or 2 or 3, got {}".format(order))

    def multistep_dpm_solver_update(self, x, model_prev_list, t_prev_list, t, order, solver_type='dpmsolver'):
        """Order dispatch (:932-954)."""
        self._refuse("direct", what="multistep_dpm_solver_update()")
        if order == 1:
            return self.dpm_solver_first_update(x, t_prev_list[-1], t, model_s=model_prev_list[-1])
        elif order == 2:
            return self.multistep_dpm_solver_second_update(x, model_prev_list, t_prev_list, t, solver_type=solver_type)
        elif order == 3:
            return self.multistep_dpm_solver_third_update(x, model_prev_list, t_prev_list, t, solver_type=solver_type)
        else:
            raise ValueError("Solver order must be 1 or 2 or 3, got {}".format(order))

    # -- adaptive solver (:956-1010) ---------------------------------------------------------------
    def dpm_solver_adaptive(self, x, order, t_T, t_0, h_init=0.05, atol=0.0078, rtol=0.05, theta=0.9,
                            t_err=1e-5, solver_type='dpmsolver'):
        """Adaptive step size DPM-Solver-12 / -23 (:956-1010). Updates and the error estimate run on
        the fused kernels; the step-size controller is the reference's host logic."""
        self._refuse("direct", what="dpm_solver_adaptive()")
        ns = self.noise_schedule
        x = self._state(x)
        device = x.device
        if order not in (2, 3):
            raise ValueError("For adaptive step size solver, order must be 2 or 3, got {}".format(order))
        if solver_type not in ['dpmsolver', 'taylor']:
            raise ValueError("'solver_type' must be either 'dpmsolver' or 'taylor', got {}".format(solver_type))
        if self._device_controller_ok(x):
            return self._adaptive_on_device(x, order, t_T, t_0, h_init, atol, rtol, theta, t_err, solver_type)
        # host controller (schedules / options the device controller does not cover, and the CPU test executor):
        # the controller's scalars live on the host (fp32, reference op order); the network receives
        # device time labels, uploaded once per iteration
        s = t_T * torch.ones((1,))
        lambda_s = ns.marginal_lambda(s)
        lambda_0 = ns.marginal_lambda(t_0 * torch.ones_like(s))
        h = h_init * torch.ones_like(s)
        x_prev = x
        nfe = 0
        if order not in (2, 3):
            raise ValueError("For adaptive step size solver, order must be 2 or 3, got {}".format(order))
        if solver_type not in ['dpmsolver', 'taylor']:
            raise ValueError("'solver_type' must be either 'dpmsolver' or 'taylor', got {}".format(solver_type))
        while torch.abs((s - t_0)).mean() > t_err:
            t = ns.inverse_lambda(lambda_s + h)
            if order == 2:      # DPM-Solver-12 (:985-988)
                sp_low = P.SinglestepPlan(1, [P._cpu(s)], [P.first_update_coeffs(ns, self.algorithm_type, s, t)])
                sp_high = P.singlestep_second(ns, self.algorithm_type, solver_type, s, t, 0.5)
            else:               # DPM-Solver-23 (:989-992)
                sp_low = P.singlestep_second(ns, self.algorithm_type, solver_type, s, t, 1. / 3.)
                sp_high = P.singlestep_third(ns, self.algorithm_type, solver_type, s, t, 1. / 3., 2. / 3.)
            t_all = self._upload(torch.cat([tt.reshape(-1) for tt in sp_high.times]), device)
            td = [t_all[j:j + 1] for j in range(len(sp_high.times))]
            x_lower, ms = self._run_singlestep(x, sp_low, keep=True, times_dev=td[:len(sp_low.times)])
            x_higher, _ = self._run_singlestep(x, sp_high, model_s=ms[0], model_s1=ms[1] if order == 3 else None,
                                               times_dev=td)
            # E = max_b sqrt(mean(((x_higher - x_lower)/delta)^2)), delta = max(atol, rtol*max(|x_lower|,|x_prev|))
            # (:999-1001): one fused reduction launch; the accept/reject test needs E on the host (:1002)
            E = ops.backend().error_norm(x_higher, x_lower, self._state_like(x_prev, x_higher.dtype), atol, rtol)
            if self.plan_broadcast and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                # batch-sharded run: E is a max over the batch (:1001), so one 4-byte all-reduce(max) per
                # iteration makes every rank take the single-process controller's decisions (SURVEY 8e)
                E = E.reshape(1).float()
                dist.all_reduce(E, op=dist.ReduceOp.MAX)
            E = E.cpu()
            if bool(torch.isnan(E).any()):
                # the reference would reject the step, set h = NaN and spin forever (s never advances, :1002-1008)
                raise FloatingPointError("dpm_solver_adaptive: the error estimate is NaN (the network output diverged)")
            if torch.all(E <= 1.):
                x = x_higher
                s = t
                x_prev = x_lower
                lambda_s = ns.marginal_lambda(s)
            h = torch.min(theta * h * torch.float_power(E, -1. / order).float(), lambda_0 - lambda_s)
            nfe += order
        print('adaptive solver nfe', nfe)
        return x

    adaptive_controller = "device"   # "host": the reference's per-iteration host decision (one sync per iteration)
    adaptive_chunk = 4               # iterations enqueued between two reads of the device-side `done` flag

    def _device_controller_ok(self, x) -> bool:
        be = ops.backend()
        w = self._wrapped
        return (self.adaptive_controller == "device" and hasattr(be, "adaptive_controller") and x.is_cuda
                and getattr(self.noise_schedule, "schedule", None) in ops.AdaptiveController.SUPPORTED
                and not self._dynamic_thresholding        # the quantile call takes alpha_t, sigma_t by value
                and not self.reference_rounding
                and not (isinstance(w, WrappedModel) and not w.fusable)      # classifier guidance: model_fn needs host scalars
                and not torch.cuda.is_current_stream_capturing())

    def _adaptive_on_device(self, x, order, t_T, t_0, h_init, atol, rtol, theta, t_err, solver_type):
        """dpm_solver_adaptive with the controller on the device (csrc/adaptive_ctl.cu): s, lambda_s, h and the
        accept/reject decision never visit the host; every fused launch reads its scalars from the coefficient
        block the plan kernel wrote; `adaptive_chunk` iterations are enqueued per read of the `done` flag."""
        be, ns = ops.backend(), self.noise_schedule
        w = self._wrapped
        # (the network's time input differs from the label: the controller writes it next to the label)
        discrete_in = isinstance(w, WrappedModel) and w.noise_schedule.schedule in ('discrete', 'flow')
        ctl = be.adaptive_controller(ns, x.device, order=order, predict_x0=self._pp, taylor=solver_type == 'taylor',
                                     t_0=t_0, theta=theta, t_err=t_err, discrete_input=discrete_in)
        ctl.init(t_T, h_init)
        x = x.clone()                 # the committed state: overwritten in place by accepted steps
        x_prev = x.clone()
        # (a 16-bit x_T reaches the network widened to fp32 here -- same values; the by-identity hand-over of the
        # caller's own tensor at the first evaluation, `_net_input`, cannot follow a buffer that is updated in place)
        self._net_input = None
        rows = w.input_rows(x.shape[0]) if isinstance(w, WrappedModel) else x.shape[0]
        C = P.Coeffs
        if order == 2:     # DPM-Solver-12 (:985-988): coefficient blocks 0 (lower), 1 (x -> x_s1), 2 (higher)
            sp_low = P.SinglestepPlan(1, [None], [C(FORM_LIN1, 0., 0., order=1, dev=ctl.block(0))])
            sp_high = P.SinglestepPlan(2, [None, None], [C(FORM_LIN1, 0., 0., order=2, dev=ctl.block(1)),
                                                         C(ops.FORM_DIFF2, 0., 0., w0=1.0, c0_on_old=True, order=2, dev=ctl.block(2))])
        else:              # DPM-Solver-23 (:989-992): blocks 0 (x -> x_s1), 1 (lower), 2 (x -> x_s2), 3 (higher)
            sp_low = P.SinglestepPlan(2, [None, None], [C(FORM_LIN1, 0., 0., order=2, dev=ctl.block(0)),
                                                        C(ops.FORM_DIFF2, 0., 0., w0=1.0, c0_on_old=True, order=2, dev=ctl.block(1))])
            fin = C(FORM_SS3T, 0., 0., order=3, dev=ctl.block(3)) if solver_type == 'taylor' else \
                C(ops.FORM_DIFF2, 0., 0., w0=1.0, c0_on_old=True, order=3, dev=ctl.block(3))
            sp_high = P.SinglestepPlan(3, [None, None, None], [C(FORM_LIN1, 0., 0., order=3, dev=ctl.block(0)),
                                                               C(ops.FORM_DIFF2, 0., 0., w0=1.0, c0_on_old=True, order=3, dev=ctl.block(2)),
                                                               fin])
        n_high = len(sp_high.times)
        td = [ctl.time(j) for j in range(n_high)]
        tin = [ctl.input_time(j).expand(rows) for j in range(n_high)] if discrete_in else [None] * n_high
        dev_als = [_DEV] * n_high
        sharded = self.plan_broadcast and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        n_low = len(sp_low.times)
        while True:
            for _ in range(max(1, int(self.adaptive_chunk))):
                ctl.plan()
                x_lower, ms = self._run_singlestep(x, sp_low, keep=True, times_dev=td[:n_low], alsig=dev_als[:n_low],
                                                   t_inputs=tin[:n_low])
                x_higher, _ = self._run_singlestep(x, sp_high, model_s=ms[0], model_s1=ms[1] if order == 3 else None,
                                                   times_dev=td, alsig=dev_als, t_inputs=tin)
                be.error_norm(x_higher, x_lower, x_prev, atol, rtol, out=ctl.E)      # :999-1001, one fused reduction
                if sharded:
                    dist.all_reduce(ctl.E, op=dist.ReduceOp.MAX)                    # E is a max over the batch (:1001)
                ctl.decide()                                                          # :1002-1008 on the device
                ctl.select_copy(x, x_higher)
                ctl.select_copy(x_prev, x_lower)
            done, nfe, _ = ctl.read()                                                 # the chunk's only host sync
            if done == 2:
                raise FloatingPointError("dpm_solver_adaptive: the error estimate is NaN (the network output diverged)")
            if done:
                break
        print('adaptive solver nfe', nfe)
        return x

    # -- add_noise / inverse (:1012-1045) --------------------------------------------------------
    def add_noise(self, x, t, noise=None):
        """xt = alpha_t * x + sigma_t * noise for every t in `t` -> (t_size, batch, *shape)."""
        th = P._cpu(t)
        alpha_t, sigma_t = self.noise_schedule.marginal_alpha(th), self.noise_schedule.marginal_std(th)
        be = ops.backend()
        if noise is None and x.is_cuda and hasattr(be, "add_noise_philox") and th.shape[0] <= 16 \
                and x.dtype in ops.SUPPORTED_DTYPES and not torch.cuda.is_current_stream_capturing():
            # the noise never touches HBM: drawn in registers by the generator torch.randn would have used, same
            # (seed, offset) -> same values, the torch generator advanced as randn would have (csrc/philox.cu)
            xs = self._state_like(x, x.dtype)
            outs = be.add_noise_philox(xs, alpha_t.tolist(), sigma_t.tolist(), self._sdtype(x))
            return outs[0] if th.shape[0] == 1 else outs
        if noise is None:
            noise = torch.randn((th.shape[0], *x.shape), device=x.device)
        # result dtype: the reference's fp32 (t_size,1,..) coefficient tensors promote a 16-bit x to fp32 (:1026)
        sd = self._sdtype(x)
        # with a 16-bit state, fp32 noise stays fp32: alpha*x + sigma*noise is rounded to the state dtype once, as the
        # in-kernel noise path does (rounding the noise to the state dtype first would round twice)
        wd = torch.float32 if noise.dtype == torch.float32 else sd
        xs = self._state_like(x, wd)
        noise = noise.reshape((th.shape[0], *x.shape))
        outs = [ops.lincomb(xs, [self._state_like(noise[i], wd)], float(alpha_t[i]), [float(sigma_t[i])]).to(sd)
                for i in range(th.shape[0])]
        if th.shape[0] == 1:
            return outs[0]
        return torch.stack(outs)

    def inverse(self, x, steps=20, t_start=None, t_end=None, order=2, skip_type='time_uniform',
                method='multistep', lower_order_final=True, denoise_to_zero=False, solver_type='dpmsolver',
                atol=0.0078, rtol=0.05, return_intermediate=False):
        """Invert `x` from t_start (default 1/N) to t_end (default T) (:1032-1045)."""
        self._refuse("inverse")
        t_0 = 1. / self.noise_schedule.total_N if t_start is None else t_start
        t_T = self.noise_schedule.T if t_end is None else t_end
        assert t_0 > 0 and t_T > 0, "Time range needs to be greater than 0. For discrete-time DPMs, it needs to be in [1 / N, 1], where N is the length of betas array"
        return self.sample(x, steps=steps, t_start=t_0, t_end=t_T, order=order, skip_type=skip_type,
                           method=method, lower_order_final=lower_order_final, denoise_to_zero=denoise_to_zero,
                           solver_type=solver_type, atol=atol, rtol=rtol, return_intermediate=return_intermediate)

    # -- whole-loop CUDA graph (SURVEY 8f-1; no counterpart in the reference) -----------------------
    def _sde_args(self, x, eta, generator) -> float:
        """Validate sample()'s eta and generator: the run's eta for the SDE solver (0: the ODE run, nothing drawn), else
        0. ValueError before any launch or network call."""
        if self.algorithm_type != "sde-dpmsolver++":
            if eta is not None or generator is not None:
                raise ValueError("eta and generator are arguments of algorithm_type='sde-dpmsolver++', not {!r}".format(
                    self.algorithm_type))
            return 0.0
        eta = 1.0 if eta is None else eta
        if isinstance(eta, bool) or not isinstance(eta, (int, float)) or not math.isfinite(eta) or eta < 0:
            raise ValueError("eta must be a finite number >= 0, got {!r}".format(eta))
        if generator is not None:
            if not isinstance(generator, torch.Generator) or not ops.same_device(generator.device, x.device):
                raise ValueError("the generator must be a torch.Generator on x's device {}, got {!r}".format(
                    x.device, getattr(generator, "device", generator)))
        return float(eta)

    def capture(self, x_example, **sample_kwargs):
        """Capture `sample(x, **sample_kwargs)` -- the network calls included -- in ONE CUDA graph.

        Once the coefficient plan and the device tables are cached, the sampling loop performs no
        host<->device copy, no synchronisation and no collective, and every kernel takes its scalars
        by value, so the whole run is capturable whenever the network is. Returns a callable
        `g(x) -> x_0` that copies `x` into the graph's static input and replays; the returned tensor
        is the graph's static output (clone it to keep it across replays). Not available for the
        adaptive method (host-side accept/reject) or with python-side hooks that synchronise."""
        if sample_kwargs.get("method", "multistep") == "adaptive":
            raise ValueError("the adaptive solver decides on the host every iteration; it cannot be captured")
        if sample_kwargs.get("return_intermediate"):
            raise ValueError("capture() returns the final sample only")
        x_static = self._state(x_example).clone()
        self.sample(x_static, **sample_kwargs)                       # builds and caches plan + tables
        graph = torch.cuda.CUDAGraph()
        gen = sample_kwargs.get("generator")
        if gen is not None and hasattr(graph, "register_generator_state"):
            graph.register_generator_state(gen)       # SDE noise from a user generator: replays advance it
        side = torch.cuda.Stream(device=x_static.device)
        side.wait_stream(torch.cuda.current_stream(x_static.device))
        with torch.cuda.stream(side):
            self.sample(x_static, **sample_kwargs)                   # warm-up on the capture stream
            with torch.cuda.graph(graph, stream=side):
                y_static = self.sample(x_static, **sample_kwargs)
        torch.cuda.current_stream(x_static.device).wait_stream(side)

        def replay(x):
            x_static.copy_(x)
            graph.replay()
            return y_static

        replay.graph, replay.static_input, replay.static_output = graph, x_static, y_static
        return replay

    # -- sample (:1047-1245) ---------------------------------------------------------------------
    def sample(self, x, steps=20, t_start=None, t_end=None, order=2, skip_type='time_uniform',
               method='multistep', lower_order_final=True, denoise_to_zero=False, solver_type='dpmsolver',
               atol=0.0078, rtol=0.05, return_intermediate=False, eta=None, generator=None):
        """Integrate the diffusion ODE from t_start to t_end; arguments as in the reference.

        With algorithm_type="sde-dpmsolver++" the run integrates the diffusion SDE instead (SDE-DPM-Solver++, Lu et al.
        2022, arXiv:2211.01095), method='multistep' only. `eta` (finite, >= 0, default 1.0) scales the noise and
        `generator` (a torch.Generator on x's device, default: that device's default generator) draws it; passing
        either with another algorithm_type is a ValueError. Take one update s -> t with h = lambda_t - lambda_s and
        h_eta = (1 + eta)*h. The host forms every scalar in fp32 through torch CPU ops, as for "dpmsolver++", with h
        replaced by h_eta in every phi and a multiplied by exp(-eta*h):
          order 1 (LIN1):  a = (sigma_t/sigma_s)*exp(-eta*h), c0 = -(alpha_t*phi_1), phi_1 = expm1(-h_eta)
          order 2 (DIFF2): a, c0 as order 1; c1 = -(0.5*(alpha_t*phi_1)) for solver_type="dpmsolver" (midpoint),
                           alpha_t*(phi_1/h_eta + 1) for "taylor" (Heun); w0 = 1/r0 as for the ODE
          order 3 (MS3):   a, c0 as order 1; phi_2 = phi_1/h_eta + 1, phi_3 = phi_2/h_eta - 0.5, c1 = alpha_t*phi_2,
                           c2 = -(alpha_t*phi_3); w0..w3 as for the ODE
        and the noise weight cz = sigma_t*sqrt(-expm1(-2*eta*h)). Per element, in fp32 with each op rounded and no
        contraction, x_t = <the ODE form's expression> + cz*z, stored in the state dtype, where update i (1..steps)
        draws z_i = torch.empty_like(x_i, dtype=torch.float32).normal_(generator=g) at that update (row-major: the
        values of torch.randn(x.shape, generator=g); channels_last: filled in storage order). The values are
        torch's bit for bit, drawn inside the fused update launch, and the generator ends where those calls would
        leave it, in program order with every other consumer of it (a correcting_xt_fn, say). Under CUDA-graph
        capture z is drawn by torch (graph-safe) and read. denoise_to_zero returns the x0 of its final evaluation and
        draws nothing. eta=0 is the "dpmsolver++" run bit for bit and draws nothing.
        Equivalences (in the VE coordinates x/alpha, sigma/alpha): k-diffusion's sample_dpmpp_2m_sde(eta,
        solver_type) is order=2, lower_order_final=False with midpoint -> "dpmsolver" and heun -> "taylor";
        sample_dpmpp_3m_sde(eta) is order=3, solver_type="taylor", lower_order_final=False (its order-2 warm-up step
        uses the Heun phi_2); diffusers' DPMSolverMultistepScheduler(algorithm_type="sde-dpmsolver++") is eta=1.
        Thresholding, correcting_x0_fn, correcting_xt_fn, return_intermediate, every skip_type, schedule and model type,
        and the guidance forms uncond, classifier, classifier-free (scalar or per-sample scale, guidance_rescale,
        cfg_zero_star, tcfg, fdg_scales) are accepted; singlestep / adaptive methods, inverse(), the direct update
        methods, several conditions, guidance_mask, perp_neg, apg_eta, cfg_pp and reference_rounding are not."""
        options = self._options()
        if method != "multistep":
            _check_options(options, ("adaptive" if method == "adaptive" else "singlestep",), "method={!r}".format(method))
        elif order not in (1, 2):
            _check_options(options, ("order",), "order {}".format(order))
        sde_eta = self._sde_args(x, eta, generator)
        t_0 = 1. / self.noise_schedule.total_N if t_end is None else t_end
        t_T = self.noise_schedule.T if t_start is None else t_start
        assert t_0 > 0 and t_T > 0, "Time range needs to be greater than 0. For discrete-time DPMs, it needs to be in [1 / N, 1], where N is the length of betas array"
        if return_intermediate:
            assert method in ['multistep', 'singlestep', 'singlestep_fixed'], "Cannot use adaptive solver when saving intermediate values"
        if self.correcting_xt_fn is not None:
            assert method in ['multistep', 'singlestep', 'singlestep_fixed'], "Cannot use adaptive solver when correcting_xt_fn is not None"
        self._check_fdg(x)
        device = x.device
        intermediates = []
        ns = self.noise_schedule
        self._xin_pair = None
        self._rr_run = 0
        # prepared launches: the CUDA executor, no python-side x0 hook, no 16-bit reference-rounding mode
        self._prep_on = (hasattr(ops.backend(), "prepare") and not self.reference_rounding and not sde_eta
                         and (self.correcting_x0_fn is None or self._dynamic_thresholding))
        with torch.no_grad(), self._apg_scope():
            x = self._state(x)
            sd = x.dtype
            if method == 'adaptive':
                x = self.dpm_solver_adaptive(x, order=order, t_T=t_T, t_0=t_0, atol=atol, rtol=rtol,
                                             solver_type=solver_type)
                step = 0
            elif method == 'multistep':
                assert steps >= order
                if solver_type not in ['dpmsolver', 'taylor'] and order >= 2:
                    raise ValueError("'solver_type' must be either 'dpmsolver' or 'taylor', got {}".format(solver_type))
                if order not in (1, 2, 3):
                    raise ValueError("Solver order must be 1 or 2 or 3, got {}".format(order))
                key = ("multistep", steps, order, skip_type, t_T, t_0, solver_type, lower_order_final)
                cfgpp = "cfgpp" in options
                if cfgpp:
                    key = key + ("cfg_pp",)     # (the plan carries g)
                if self.algorithm_type == "sde-dpmsolver++":
                    key = key + ("eta", sde_eta)    # (the plan carries h_eta's coefficients and cz)

                def build():
                    ts = self.get_time_steps(skip_type=skip_type, t_T=t_T, t_0=t_0, N=steps, device='cpu')
                    assert ts.shape[0] - 1 == steps
                    marg = P.Marginals(ns, ts)
                    plan = P.multistep_plan(ns, "dpmsolver++" if self._pp else self.algorithm_type, solver_type, ts,
                                            order, lower_order_final, marginals=marg, cfg_pp=cfgpp, eta=sde_eta)
                    # (alpha_t, sigma_t) per grid point: scalars of the eps->x0 / parameterisation step
                    return ts, plan, list(zip(marg.alpha_e.tolist(), marg.sigma.tolist()))

                ts, plan, alsig = self._host_plan(key, build)
                plan = self._sync_plan(plan, key)
                _, _, ts_dev, _, tin = self._device_tables(key, ts, x.shape[0], device)   # lists of per-step views
                # model evaluation 0, then one fused launch per step:
                #   m_{i} = convert(net(x_i, t_i));  x_{i+1} = update(x_i, m_i, m_{i-1}, m_{i-2})
                step = 0
                pid = self._plan_id(key)
                raw = self._evaluate(x, ts_dev[0], None if tin is None else tin[0])
                xe = x
                if self.correcting_xt_fn is not None:
                    x = self._state_like(self.correcting_xt_fn(x, ts_dev[0], step), sd)
                if return_intermediate:
                    intermediates.append(x)
                older: List[torch.Tensor] = []  # buffered model values, newest last
                for step in range(1, steps + 1):
                    co = plan[step - 1]
                    m1 = older[-1] if co.order >= 2 else None
                    m2 = older[-2] if co.order >= 3 else None
                    want = order >= 2 and step < steps
                    if sde_eta:
                        # the update launch of this step adds cz*z, its noise drawn at that launch
                        self._sde_noise = ops.SdeNoise(co.cz, generator)
                    try:
                        m_new, x_new = self._post_model(raw, xe, ts_dev[step - 1], alsig[step - 1], co, x,
                                                        m1, m2, want_m=want, dup_out=step < steps,
                                                        slot=(pid, step))
                    finally:
                        self._sde_noise = None
                    x = x_new
                    t = ts_dev[step]
                    if self.correcting_xt_fn is not None:
                        x = self._state_like(self.correcting_xt_fn(x, t, step), sd)
                    if return_intermediate:
                        intermediates.append(x)
                    if m_new is not None:
                        older.append(m_new)
                        if len(older) > 2:
                            older.pop(0)
                    # We do not need to evaluate the final model value.
                    if step < steps:
                        raw = self._evaluate(x, t, None if tin is None else tin[step])
                        xe = x
            elif method in ['singlestep', 'singlestep_fixed']:
                key = (method, steps, order, skip_type, t_T, t_0, solver_type)

                def build():
                    if method == 'singlestep':
                        timesteps_outer, orders = self.get_orders_and_timesteps_for_singlestep_solver(
                            steps=steps, order=order, skip_type=skip_type, t_T=t_T, t_0=t_0, device='cpu')
                    else:
                        K = steps // order
                        orders = [order, ] * K
                        timesteps_outer = self.get_time_steps(skip_type=skip_type, t_T=t_T, t_0=t_0, N=K, device='cpu')
                    if solver_type not in ['dpmsolver', 'taylor'] and max(orders) >= 2:
                        raise ValueError("'solver_type' must be either 'dpmsolver' or 'taylor', got {}".format(solver_type))
                    # host plan for the whole run (:1221-1228 evaluated up front, no .item() syncs later)
                    plans = []
                    for i, o in enumerate(orders):
                        s_, t_ = timesteps_outer[i], timesteps_outer[i + 1]
                        timesteps_inner = self.get_time_steps(skip_type=skip_type, t_T=s_.item(), t_0=t_.item(), N=o, device='cpu')
                        lambda_inner = ns.marginal_lambda(timesteps_inner)
                        h = lambda_inner[-1] - lambda_inner[0]
                        r1 = None if o <= 1 else (lambda_inner[1] - lambda_inner[0]) / h
                        r2 = None if o <= 2 else (lambda_inner[2] - lambda_inner[0]) / h
                        plans.append(P.singlestep_plan(ns, self.algorithm_type, solver_type, o, s_, t_, r1, r2))
                    if not plans:
                        # steps < order with 'singlestep_fixed': K = 0, the reference runs no outer step (:1216-1220)
                        return timesteps_outer.reshape(-1), plans, []
                    all_times = torch.cat([tt.reshape(-1) for sp in plans for tt in sp.times])
                    marg = P.Marginals(ns, all_times)
                    return (torch.cat([all_times, timesteps_outer.reshape(-1)]), plans,
                            list(zip(marg.alpha_e.tolist(), marg.sigma.tolist())))

                packed, plans, alsig = self._host_plan(key, build)
                if self.plan_broadcast and plans:
                    flat = self._sync_plan([co for sp in plans for co in sp.stages], key)
                    plans = [P.SinglestepPlan(sp.order, sp.times, []) for sp in plans]
                    k = 0
                    for sp in plans:
                        n_st = {1: 1, 2: 2, 3: 3}[sp.order]
                        sp.stages = flat[k:k + n_st]
                        k += n_st
                n_eval = len(alsig)
                _, _, _, packed1, tin = self._device_tables(key, packed, x.shape[0], device, n_eval) if plans \
                    else (None, None, None, None, None)
                all_dev, outer_dev = (packed1[:n_eval], packed1[n_eval:]) if plans else (None, None)
                k = 0
                step = 0
                pid = self._plan_id(key)
                for step, sp in enumerate(plans):
                    nt = len(sp.times)
                    td = all_dev[k:k + nt]
                    x, _ = self._run_singlestep(x, sp, times_dev=td, alsig=alsig[k:k + nt],
                                                t_inputs=None if tin is None else tin[k:k + nt],
                                                dup_last=step + 1 < len(plans), slot=(pid, step))
                    k += nt
                    if self.correcting_xt_fn is not None:
                        x = self._state_like(self.correcting_xt_fn(x, outer_dev[step + 1].reshape(()), step), sd)
                    if return_intermediate:
                        intermediates.append(x)
            else:
                raise ValueError("Got wrong method {}".format(method))
            if denoise_to_zero:
                # :1236-1238. The label, its model-input time and (alpha, sigma) at t_0 are cached with the tables:
                # no host<->device traffic in the steady state, so the tail is CUDA-graph capturable too
                t, tin0, als0 = self._denoise_tables(t_0, x.shape[0], device)
                xs = self._state(x)
                x = self._post_model(self._evaluate(xs, t, tin0), xs, t, als0, x0=True)[0]
                if self.correcting_xt_fn is not None:
                    x = self.correcting_xt_fn(x, t, step + 1)
                if return_intermediate:
                    intermediates.append(x)
        self._net_input = None
        if return_intermediate:
            return x, intermediates
        else:
            return x
