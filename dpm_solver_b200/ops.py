"""Tensor-level front end of the C-ABI: one call = one fused kernel launch on the current stream.

`StepArgs` mirrors `struct dpm_step_desc` (include/dpm_solver_b200.h) with torch tensors in place
of raw pointers. The only executor shipped is `CudaBackend`, which hands device pointers to
libdpmsolver_b200.so; it refuses CPU tensors (there is no CPU or PyTorch fallback).  Tests may
install another executor with `set_backend()` to exercise the host-side logic without a GPU.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from dataclasses import dataclass
import math
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import (DPM_BF16, DPM_F16, DPM_F32, FORM_DIFF2, FORM_LIN1, FORM_LIN2, FORM_LIN3,
                   FORM_MS3, FORM_NONE, FORM_SS3T, PARAM_NOISE, StepDesc)

_DTYPE_CODE = {torch.float32: DPM_F32, torch.bfloat16: DPM_BF16, torch.float16: DPM_F16}
SUPPORTED_DTYPES = tuple(_DTYPE_CODE)


@dataclass
class StepArgs:
    """One fused solver step (see dpm_step_desc for the meaning of every field)."""
    form: int = FORM_NONE
    n_model: int = 0
    x: Optional[torch.Tensor] = None
    xe: Optional[torch.Tensor] = None
    m0: Optional[torch.Tensor] = None
    m1: Optional[torch.Tensor] = None
    m2: Optional[torch.Tensor] = None
    e_cond: Optional[torch.Tensor] = None
    e_uncond: Optional[torch.Tensor] = None
    thr: Optional[torch.Tensor] = None
    per_sample: int = 0
    param: int = PARAM_NOISE
    predict_x0: bool = False
    c0_on_old: bool = False
    guidance: float = 1.0
    alpha_e: float = 1.0
    sigma_e: float = 0.0
    a: float = 0.0
    c0: float = 0.0
    c1: float = 0.0
    c2: float = 0.0
    w0: float = 0.0
    w1: float = 0.0
    w2: float = 0.0
    w3: float = 0.0
    w4: float = 0.0
    want_m_out: bool = False          # materialise the computed model value (n_model >= 1)
    state_dtype: Optional[torch.dtype] = None  # dtype of x/xe/m*/outputs; default: from tensors
    out: Optional[torch.Tensor] = None     # optional preallocated outputs
    out2: Optional[torch.Tensor] = None    # optional second copy of x_t (doubled CFG batch)
    m_out: Optional[torch.Tensor] = None
    raw_round: int = 0                # reference-rounding mode (dpm_step_desc.raw_round); 0 = off
    coef_dev: Optional[torch.Tensor] = None   # 16 fp32 on the device: the launch reads its scalars there (dev_coef)
    # guidance rescale (dpm_step_rescaled; n_model == 2, per_sample set): fp32 [B] from cfg_rescale_ratio, and phi
    ratio: Optional[torch.Tensor] = None
    phi: float = 0.0
    # per-sample classifier-free guidance (dpm_step_guided; n_model == 2, per_sample set): fp32 [B] on the device, in
    # place of `guidance`. With `ratio` the step is also rescaled.
    guidance_b: Optional[torch.Tensor] = None
    # multi-condition classifier-free guidance (dpm_step_multi; n_model == 2): the K >= 2 conditional outputs, in place
    # of `e_cond` (which holds the first of them), their K fp32-rounded python-float scales, in place of `guidance`, and
    # optionally K tensors that receive x_t again (blocks 1..K of the next network input; `out2` is not used)
    e_conds: Optional[Tuple[torch.Tensor, ...]] = None
    scales: Optional[Tuple[float, ...]] = None
    replicas: Optional[Tuple[torch.Tensor, ...]] = None
    # regional guidance (dpm_step_multi_masked; with e_conds, 1 <= K <= 4, per_sample set): one weight map per condition,
    # None (all ones), (w, period, sample_stride) with w a contiguous fp32 tensor on the tensors' device, or an object
    # whose weights(shape, layout, device) gives that triple for the launch's shape and storage order ('c' or 'cl'). The
    # weight of scales[k] at element i (storage order) is w.view(-1)[b*sample_stride + (i - b*per_sample) % period],
    # b = i // per_sample.
    masks: Optional[Tuple[Optional[tuple], ...]] = None
    # UniPC (dpm_step_unipc): the launch's words (plan.UniCoeffs), m_{i-3}, and an optional preallocated tensor that
    # receives the corrected state x_i (required when the launch has no predictor). `x` is x~_i, `m1`/`m2` m_{i-1}/m_{i-2}.
    unipc: Optional[object] = None
    m3: Optional[torch.Tensor] = None
    out_c: Optional[torch.Tensor] = None
    # adaptive projected guidance (dpm_step_apg; n_model == 2, per_sample set): the words [2, B] of `apg_words()`, the
    # fp32 direction R it wrote (read in place of `e_uncond`; None: R from e_uncond), and the marginals of the x0 -> eps
    # conversion of an eps step. `alpha_e`, `sigma_e` are those of the x0 conversion (EDM: its x0 words); `guidance_b`,
    # when set, gives the per-sample scales (a scale of 1 bypasses).
    apg_words: Optional[torch.Tensor] = None
    apg_r: Optional[torch.Tensor] = None
    alpha_t: float = 1.0
    sigma_t: float = 0.0
    # CFG-Zero* (dpm_step_cfgzero; n_model == 2, per_sample set): the per-sample scales s* of `cfgzero_scale()`, fp32
    # [B]; `guidance_b`, when set, gives the per-sample guidance scales (else `guidance`)
    cfgzero_s: Optional[torch.Tensor] = None
    # TCFG (dpm_step_tcfg; n_model == 2, per_sample set): the per-sample words (wu, wc) of `tcfg_words()`, fp32 [B, 2];
    # `guidance_b`, when set, gives the per-sample guidance scales (else `guidance`)
    tcfg_w: Optional[torch.Tensor] = None
    # CFG++ (dpm_step_cfgpp; form LIN1 or DIFF2, n_model == 2, predict_x0): alpha_t of the update's end time, the weight
    # of G - U; None is off. m_out then receives U, the x0 of e_uncond alone; `guidance_b`, when set, gives the
    # per-sample scales (else `guidance`, always combined)
    cfgpp_g: Optional[float] = None
    # SDE-DPM-Solver++ (dpm_step_sde; form LIN1, DIFF2 or MS3): the update's Gaussian noise, None is off
    sde: Optional["SdeNoise"] = None

    def state_tensors(self):
        return [t for t in (self.x, self.xe, self.m0, self.m1, self.m2) if t is not None]

    def model_tensors(self):
        return [t for t in (self.e_cond, self.e_uncond) if t is not None]

    def reference_tensor(self) -> torch.Tensor:
        for t in (self.x, self.xe, self.e_cond, self.m0):
            if t is not None:
                return t
        raise ValueError("StepArgs without tensors")


@dataclass
class SdeNoise:
    """The noise of one SDE-DPM-Solver++ update: out = <the update> + cz*z, z = torch.empty_like(x,
    dtype=torch.float32).normal_(generator=generator) drawn at the launch (generator None: the default generator of x's
    device), in x's storage order."""
    cz: float
    generator: Optional[torch.Generator] = None


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
if _raw_stream is None:  # older torch: go through the Stream object
    def _raw_stream(idx):
        return torch.cuda.current_stream(idx).cuda_stream


def fdg_check(shape, levels: int, dtype=torch.float32) -> None:
    """ValueError unless frequency-decoupled guidance serves outputs of `shape` with `levels` levels: at least 4 dims,
    and planes of the last two that dpm_fdg_supported accepts (the library's one statement of the size rule)."""
    if len(shape) < 4:
        raise ValueError("frequency-decoupled guidance needs x with at least 4 dims [B, C, ..., H, W], got shape "
                         "{}".format(tuple(shape)))
    if dtype not in _DTYPE_CODE:
        raise TypeError("dpm_solver_b200: unsupported dtype {} for frequency-decoupled guidance".format(dtype))
    lib = _lib.lib()
    if lib.dpm_fdg_supported(int(shape[-2]), int(shape[-1]), int(levels), _DTYPE_CODE[dtype]) != 0:
        raise ValueError("frequency-decoupled guidance with x of shape {}: {}".format(
            tuple(shape), lib.dpm_last_error().decode("utf-8", "replace")))


def same_device(a: torch.device, b: torch.device) -> bool:
    """One device, a CUDA device without an index meaning the current one (torch.Generator("cuda") reports none)."""
    if a.type != b.type:
        return False
    if a.type != "cuda":
        return True
    cur = torch.cuda.current_device() if (a.index is None or b.index is None) else None
    return (cur if a.index is None else a.index) == (cur if b.index is None else b.index)


def _dense(t: torch.Tensor) -> bool:
    """True when the elements of `t` fill its storage span exactly once in some order of its dims (row-major,
    channels_last, transposed or otherwise permuted views): an output allocated with its strides has no gaps."""
    expect = 1
    for st, n in sorted((st, n) for n, st in zip(t.shape, t.stride()) if n != 1):
        if st != expect:
            return False
        expect *= n
    return True


def _plane_strides(t: torch.Tensor):
    """(sample_stride, plane_stride, h_stride, w_stride) in elements of a [B, *mid, H, W] tensor whose planes are
    indexed by one stride over the flattened mid dims (row-major and 4-D channels_last alike), else None."""
    mid = [(n, st) for n, st in zip(t.shape[1:-2], t.stride()[1:-2]) if n != 1]
    for (n0, s0), (n1, s1) in zip(mid, mid[1:]):
        if s0 != s1 * n1:
            return None
    plane = mid[-1][1] if mid else 0
    return t.stride(0), plane, t.stride(-2), t.stride(-1)


class CudaBackend:
    """Executes StepArgs through libdpmsolver_b200.so."""

    name = "cuda-sm90a"

    def __init__(self):
        self._lib = _lib.lib()  # fail loudly at construction if the .so is missing

    # -- helpers --------------------------------------------------------------------------
    @staticmethod
    def _layout(t: torch.Tensor) -> Optional[str]:
        """'c' (row-major dense), 'cl' (channels_last dense) or None (needs a copy). Element-wise
        kernels only need every operand to share ONE dense layout: the storage is then a flat array."""
        if t.is_contiguous():
            return "c"
        if t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last):
            return "cl"
        if t.dim() == 5 and t.is_contiguous(memory_format=torch.channels_last_3d):
            return "cl"
        return None

    @staticmethod
    def _check(t: torch.Tensor, what: str, dev, numel: int, dtype=None, layout: str = "c") -> torch.Tensor:
        if not t.is_cuda:
            raise RuntimeError(f"dpm_solver_b200: `{what}` is on {t.device}; this library is CUDA-only "
                               "(no CPU fallback)")
        if t.device != dev:
            raise RuntimeError(f"dpm_solver_b200: `{what}` is on {t.device}, expected {dev}")
        if t.numel() != numel:
            raise ValueError(f"dpm_solver_b200: `{what}` has {t.numel()} elements, expected {numel}")
        if dtype is not None and t.dtype != dtype:
            raise TypeError(f"dpm_solver_b200: `{what}` is {t.dtype}, expected {dtype}")
        if t.dtype not in _DTYPE_CODE:
            raise TypeError(f"dpm_solver_b200: unsupported dtype {t.dtype} for `{what}`")
        if layout == "cl":
            if t.dim() in (4, 5) and t.is_contiguous(memory_format=torch.channels_last if t.dim() == 4 else torch.channels_last_3d):
                return t
            return t.contiguous(memory_format=torch.channels_last if t.dim() == 4 else torch.channels_last_3d) \
                if t.dim() in (4, 5) else t.contiguous()
        return t if t.is_contiguous() else t.contiguous()

    def _fill(self, a: StepArgs):
        ref = a.reference_tensor()
        dev, n = ref.device, ref.numel()
        sdt = a.state_dtype
        if sdt is None:
            st = a.state_tensors()
            sdt = st[0].dtype if st else a.e_cond.dtype
        # channels_last networks hand over channels_last tensors: keep that layout end to end
        layout = self._layout(ref) or "c"
        for t in (a.out, a.m_out, a.out2):
            if t is not None and self._layout(t) != layout:
                layout = "c"   # preallocated row-major outputs: bring the inputs to that layout
        keep = []  # keep converted copies alive until after the launch
        d = StepDesc()

        def ptr(t, what, dtype):
            if t is None:
                return None
            t = self._check(t, what, dev, n, dtype, layout)
            keep.append(t)
            return t.data_ptr()

        d.x = ptr(a.x, "x", sdt)
        d.xe = ptr(a.xe, "xe", sdt)
        d.m0 = ptr(a.m0, "m0", sdt)
        d.m1 = ptr(a.m1, "m1", sdt)
        d.m2 = ptr(a.m2, "m2", sdt)
        mdt = a.e_cond.dtype if a.e_cond is not None else sdt
        d.e_cond = ptr(a.e_cond, "e_cond", mdt)
        d.e_uncond = ptr(a.e_uncond, "e_uncond", mdt)
        if a.thr is not None:
            if not a.thr.is_cuda or a.thr.dtype != torch.float32 or not a.thr.is_contiguous():
                raise TypeError("dpm_solver_b200: `thr` must be a contiguous fp32 CUDA tensor")
            if a.per_sample <= 0 or n % a.per_sample or a.thr.numel() != n // a.per_sample:
                raise ValueError("dpm_solver_b200: `thr` needs one value per sample")
            keep.append(a.thr)
            d.thr = a.thr.data_ptr()
        d.n = n
        d.per_sample = a.per_sample
        d.state_dtype = _DTYPE_CODE[sdt]
        d.model_dtype = _DTYPE_CODE[mdt]
        d.form, d.n_model, d.param = a.form, a.n_model, a.param
        d.predict_x0, d.c0_on_old = int(a.predict_x0), int(a.c0_on_old)
        d.raw_round = int(a.raw_round)
        d.guidance, d.alpha_e, d.sigma_e = a.guidance, a.alpha_e, a.sigma_e
        d.a, d.c0, d.c1, d.c2 = a.a, a.c0, a.c1, a.c2
        d.w0, d.w1, d.w2, d.w3, d.w4 = a.w0, a.w1, a.w2, a.w3, a.w4
        if a.coef_dev is not None:
            cd = a.coef_dev
            if not cd.is_cuda or cd.dtype != torch.float32 or cd.numel() < 16 or not cd.is_contiguous() or cd.device != dev:
                raise TypeError("dpm_solver_b200: `coef_dev` must be 16 contiguous fp32 values on the tensors' device")
            keep.append(cd)
            d.dev_coef = cd.data_ptr()
        return d, keep, ref, sdt, layout

    def _new_like(self, ref, sdt, layout):
        if layout == "cl":
            return torch.empty(ref.shape, dtype=sdt, device=ref.device,
                               memory_format=torch.channels_last if ref.dim() == 4 else torch.channels_last_3d)
        return torch.empty(ref.shape, dtype=sdt, device=ref.device)

    # -- API -----------------------------------------------------------------------------
    def step(self, a: StepArgs) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """Launch one fused step. Returns (m_out, out); either may be None."""
        d, keep, ref, sdt, layout = self._fill(a)
        m_out = out = None
        if a.n_model > 0 and (a.want_m_out or a.form == FORM_NONE):
            m_out = a.m_out if a.m_out is not None else self._new_like(ref, sdt, layout)
            self._check(m_out, "m_out", ref.device, ref.numel(), sdt)
            if self._layout(m_out) != layout:
                raise ValueError("dpm_solver_b200: preallocated m_out must be dense and laid out like the inputs")
            d.m_out = m_out.data_ptr()
        if a.form != FORM_NONE and (a.unipc is None or a.unipc.pp > 0):
            out = a.out if a.out is not None else self._new_like(ref, sdt, layout)
            self._check(out, "out", ref.device, ref.numel(), sdt)
            if self._layout(out) != layout:
                raise ValueError("dpm_solver_b200: preallocated out must be dense and laid out like the inputs")
            d.out = out.data_ptr()
            if a.out2 is not None:
                self._check(a.out2, "out2", ref.device, ref.numel(), sdt)
                if self._layout(a.out2) != layout:      # dense, laid out like `out` (a channels_last half of the
                    raise ValueError("dpm_solver_b200: out2 must be dense and laid out like out")   # doubled CFG batch is)
                d.out2 = a.out2.data_ptr()
        self._check_per_sample(a, ref)
        if a.sde is not None:
            self._step_sde(a, d, ref, layout, keep)
        elif a.unipc is not None:
            self._step_unipc(a, d, ref, sdt, layout, keep)
        elif a.e_conds is not None:
            self._step_multi(a, d, ref, sdt, layout, keep)
        elif a.apg_words is not None:
            r = None
            if a.apg_r is not None:
                r = self._check(a.apg_r, "apg_r", ref.device, ref.numel(), torch.float32, layout)
                keep.append(r)
            self._launch(ref.device, self._lib.dpm_step_apg, C.byref(d), C.c_void_p(a.apg_words.data_ptr()),
                         C.c_void_p(None if a.guidance_b is None else a.guidance_b.data_ptr()),
                         C.c_void_p(None if r is None else r.data_ptr()), C.c_float(a.alpha_t), C.c_float(a.sigma_t))
        elif a.cfgpp_g is not None:
            if a.thr is not None or a.ratio is not None or a.cfgzero_s is not None or a.tcfg_w is not None:
                raise ValueError("dpm_solver_b200: a CFG++ step takes one or per-sample scales, without thresholds, "
                                 "rescale, CFG-Zero* or TCFG")
            self._launch(ref.device, self._lib.dpm_step_cfgpp, C.byref(d), C.c_float(a.cfgpp_g),
                         C.c_void_p(None if a.guidance_b is None else a.guidance_b.data_ptr()))
        elif a.cfgzero_s is not None:
            if a.tcfg_w is not None:
                raise ValueError("dpm_solver_b200: a step takes CFG-Zero* scales or TCFG words, not both")
            self._launch(ref.device, self._lib.dpm_step_cfgzero, C.byref(d), C.c_void_p(a.cfgzero_s.data_ptr()),
                         C.c_void_p(None if a.guidance_b is None else a.guidance_b.data_ptr()))
        elif a.tcfg_w is not None:
            if a.ratio is not None:
                raise ValueError("dpm_solver_b200: a TCFG step takes no rescale")
            self._launch(ref.device, self._lib.dpm_step_tcfg, C.byref(d), C.c_void_p(a.tcfg_w.data_ptr()),
                         C.c_void_p(None if a.guidance_b is None else a.guidance_b.data_ptr()))
        elif a.guidance_b is not None:
            # (phi and 1 - phi as below; ignored without a ratio)
            self._launch(ref.device, self._lib.dpm_step_guided, C.byref(d), C.c_void_p(a.guidance_b.data_ptr()),
                         C.c_void_p(None if a.ratio is None else a.ratio.data_ptr()), C.c_float(a.phi),
                         C.c_float(1.0 - a.phi))
        elif a.ratio is not None:
            # phi and 1 - phi (formed in double, as the python-float expression does), each rounded to fp32 once
            self._launch(ref.device, self._lib.dpm_step_rescaled, C.byref(d), C.c_void_p(a.ratio.data_ptr()),
                         C.c_float(a.phi), C.c_float(1.0 - a.phi))
        else:
            self._launch(ref.device, self._lib.dpm_step, C.byref(d))
        return m_out, out

    @staticmethod
    def _check_per_sample(a: StepArgs, ref) -> None:
        """The per-sample operands of a step: fp32 on the tensors' device, one value per sample (the APG words two)."""
        for v, what, k in ((a.ratio, "ratio", 1), (a.guidance_b, "guidance_b", 1), (a.apg_words, "apg_words", 2),
                           (a.cfgzero_s, "cfgzero_s", 1), (a.tcfg_w, "tcfg_w", 2)):
            if v is None:
                continue
            if not v.is_cuda or v.dtype != torch.float32 or not v.is_contiguous() or v.device != ref.device:
                raise TypeError(f"dpm_solver_b200: `{what}` must be a contiguous fp32 tensor on the tensors' device")
            if a.per_sample <= 0 or ref.numel() % a.per_sample or v.numel() != k * (ref.numel() // a.per_sample):
                raise ValueError(f"dpm_solver_b200: `{what}` needs {k} value(s) per sample")

    def apg_words(self, a: StepArgs, eta: float, norm_threshold: float, momentum: float,
                  r_prev: Optional[torch.Tensor] = None, r_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The per-sample words (A, B) of adaptive projected guidance as fp32 [2, B] on the device (dpm_apg_words), from
        the CFG pair, conversion and scale(s) of `a` (a.guidance_b: per-sample scales). R = D, or D + momentum*r_prev
        when r_prev is given; r_out (fp32, laid out like the outputs, may be r_prev) receives R."""
        d, keep, ref, _, layout = self._fill(a)
        if a.n_model != 2 or a.per_sample <= 0 or ref.numel() % a.per_sample:
            raise ValueError("dpm_solver_b200: the APG words take a CFG pair (n_model == 2) and per_sample")
        nb = ref.numel() // a.per_sample
        self._check_per_sample(dataclasses.replace(a, apg_words=None), ref)
        rp = ro = None
        if r_prev is not None:
            rp = self._check(r_prev, "r_prev", ref.device, ref.numel(), torch.float32, layout)
            keep.append(rp)
        if r_out is not None:
            self._check(r_out, "r_out", ref.device, ref.numel(), torch.float32)
            if self._layout(r_out) != layout:
                raise ValueError("dpm_solver_b200: r_out must be dense and laid out like the inputs")
            ro = r_out
        words = torch.empty(2, nb, dtype=torch.float32, device=ref.device)
        ws, ws_bytes = self._workspace(self._lib.dpm_apg_workspace, nb, a.per_sample, ref.device)
        self._launch(ref.device, self._lib.dpm_apg_words, C.c_void_p(words.data_ptr()), C.byref(d),
                     C.c_void_p(None if a.guidance_b is None else a.guidance_b.data_ptr()), C.c_float(eta),
                     C.c_float(norm_threshold), C.c_float(momentum), C.c_void_p(None if rp is None else rp.data_ptr()),
                     C.c_void_p(None if ro is None else ro.data_ptr()), C.c_void_p(ws.data_ptr()), C.c_size_t(ws_bytes))
        return words

    def cfgzero_scale(self, e_cond: torch.Tensor, e_uncond: torch.Tensor) -> torch.Tensor:
        """CFG-Zero*'s per-sample s*_b = <c_b, u_b> / (||u_b||^2 + 1e-8) of the two raw halves, as fp32 [B] on the
        device (dpm_cfgzero_scale): fp64 sums in storage order, merged per chunk in order. Both halves keep a shared
        dense layout (a sample is one contiguous block in row-major and channels_last storage alike)."""
        return self._words(self._lib.dpm_cfgzero_scale, self._lib.dpm_cfgzero_workspace, (),
                           [("e_cond", e_cond), ("e_uncond", e_uncond)], lambda p, ps, n, dt: (*p, dt, ps, n))

    def tcfg_words(self, e_cond: torch.Tensor, e_uncond: torch.Tensor) -> torch.Tensor:
        """TCFG's per-sample words (wu_b, wc_b), u' = wu_b*u + wc_b*c the projection of the unconditional output on the
        first right singular vector of [u_b; c_b], as fp32 [B, 2] on the device (dpm_tcfg_words): fp64 sums ||u||^2,
        <u, c>, ||c||^2 in storage order, merged per chunk in order, then the closed form of the header. Both halves
        keep a shared dense layout (a sample is one contiguous block in row-major and channels_last storage alike)."""
        return self._words(self._lib.dpm_tcfg_words, self._lib.dpm_tcfg_workspace, (2,),
                           [("e_cond", e_cond), ("e_uncond", e_uncond)], lambda p, ps, n, dt: (*p, dt, ps, n))

    def perpneg_words(self, e_uncond: torch.Tensor, e_conds, scales) -> torch.Tensor:
        """Perp-Neg's per-sample weight of the first condition, w_1 = fl32(s_1 - sum_{k>=2} s_k*<d_k, d_1>/||d_1||^2)
        with d_k = e_k - u, as fp32 [B] on the device (dpm_perpneg_words): fp64 sums in storage order, merged per chunk
        in order, then the header's left-to-right fp64 fold. `scales`: the K python-float scales (fp32-rounded). All
        K+1 blocks keep a shared dense layout (a sample is one contiguous block in row-major and channels_last storage
        alike)."""
        K = len(e_conds)
        if not 2 <= K <= _lib.MAX_CONDITIONS or len(scales) != K:
            raise ValueError("dpm_solver_b200: Perp-Neg words take 2..{} conditional outputs and one scale each".format(
                _lib.MAX_CONDITIONS))
        blocks = [("e_uncond", e_uncond)] + [("e_conds[%d]" % k, e) for k, e in enumerate(e_conds)]
        return self._words(self._lib.dpm_perpneg_words, self._lib.dpm_perpneg_workspace, (), blocks,
                           lambda p, ps, n, dt: (p[0], (C.c_void_p * K)(*p[1:]), (C.c_float * K)(*scales), C.c_int(K),
                                                 dt, ps, n))

    def _words(self, fn, workspace, shape, blocks, args):
        """Launch the words pass fn(out, *args(pointers, per_sample, n, dtype), ws, ws_bytes) over the [B, ...] network
        output blocks, given as (name, tensor), and return its fp32 words [B, *shape]. The blocks keep a shared dense
        layout (a sample is one contiguous block in row-major and channels_last storage alike), else all go row-major;
        all take the first block's device and dtype. `args` gets the ctypes values of the blocks' data pointers,
        per_sample, n and the dtype code."""
        ref = blocks[0][1]
        n, dev = ref.numel(), ref.device
        layout = self._layout(ref)
        if layout is None or any(self._layout(t) != layout for _, t in blocks):
            layout = "c"
        ts = [self._check(t, what, dev, n, None if k == 0 else ref.dtype, layout) for k, (what, t) in enumerate(blocks)]
        nb = ref.shape[0]
        per_sample = n // nb
        out = torch.empty(nb, *shape, dtype=torch.float32, device=dev)
        ws, ws_bytes = self._workspace(workspace, nb, per_sample, dev)
        middle = args([C.c_void_p(t.data_ptr()) for t in ts], C.c_uint64(per_sample), C.c_uint64(n),
                      C.c_int(_DTYPE_CODE[ref.dtype]))
        self._launch(dev, fn, C.c_void_p(out.data_ptr()), *middle, C.c_void_p(ws.data_ptr()), C.c_size_t(ws_bytes))
        return out

    @staticmethod
    def _workspace(workspace, n_samples, per_sample, dev):
        """The device workspace of a words pass (at least 8 bytes, so that it has an address) and its size."""
        ws_bytes = int(workspace(n_samples, per_sample))
        return torch.empty(max(ws_bytes, 8), dtype=torch.uint8, device=dev), ws_bytes

    def fdg_guided(self, e_cond: torch.Tensor, e_uncond: torch.Tensor, scales, levels: int) -> torch.Tensor:
        """Frequency-decoupled guidance (dpm_fdg_guided, one launch): g over the planes of the last two dims, in the
        outputs' dtype and dense layout. `scales`: `levels` python floats shared by the batch, or an fp32 [B, levels]
        tensor on the outputs' device (one row per sample)."""
        dev = e_cond.device
        fdg_check(e_cond.shape, levels, e_cond.dtype)
        for t, what in ((e_cond, "e_cond"), (e_uncond, "e_uncond")):
            if not t.is_cuda or t.device != dev:
                raise RuntimeError(f"dpm_solver_b200: `{what}` is on {t.device}; expected {dev} (CUDA only)")
            if t.dtype != e_cond.dtype or t.shape != e_cond.shape:
                raise ValueError(f"dpm_solver_b200: `{what}` is {t.dtype} {tuple(t.shape)}, expected "
                                 f"{e_cond.dtype} {tuple(e_cond.shape)}")
        ec, eu = e_cond, e_uncond
        strides = _plane_strides(ec) if _dense(ec) else None
        if strides is None or eu.stride() != ec.stride():
            ec, eu = ec.contiguous(), eu.contiguous()       # (any other layout: the same bits, at a copy's cost)
            strides = _plane_strides(ec)
        g = torch.empty_strided(ec.shape, ec.stride(), dtype=ec.dtype, device=dev)
        B, H, W = ec.shape[0], ec.shape[-2], ec.shape[-1]
        pps = math.prod(ec.shape[1:-2])
        if torch.is_tensor(scales):
            if not scales.is_cuda or scales.device != dev or scales.dtype != torch.float32 \
                    or tuple(scales.shape) != (B, levels) or not scales.is_contiguous():
                raise ValueError("dpm_solver_b200: per-sample FDG scales must be a contiguous fp32 [{}, {}] tensor on "
                                 "{}".format(B, levels, dev))
            sp, stride = C.c_void_p(scales.data_ptr()), levels
        else:
            host = (C.c_float * levels)(*scales)
            sp, stride = C.cast(host, C.c_void_p), 0
        self._launch(dev, self._lib.dpm_fdg_guided, C.c_void_p(g.data_ptr()), C.c_void_p(ec.data_ptr()),
                     C.c_void_p(eu.data_ptr()), C.c_int(_DTYPE_CODE[ec.dtype]), C.c_uint64(B * pps), C.c_uint64(H),
                     C.c_uint64(W), *(C.c_int64(v) for v in strides), C.c_int(levels), sp, C.c_uint64(stride),
                     C.c_uint64(pps))
        return g

    def _step_multi(self, a: StepArgs, d, ref, sdt, layout, keep) -> None:
        """dpm_step_multi: the K conditional outputs and scales of a multi-condition CFG step (d already filled); with
        `a.masks`, dpm_step_multi_masked (1 <= K <= 4)."""
        K = len(a.e_conds)
        k_min = 1 if a.masks is not None else 2
        if not k_min <= K <= _lib.MAX_CONDITIONS or a.scales is None or len(a.scales) != K or a.n_model != 2 \
                or a.masks is not None and len(a.masks) != K:
            raise ValueError("dpm_solver_b200: a multi-condition step takes {}..{} conditional outputs, one scale (and "
                             "with masks one mask) each, and n_model == 2".format(k_min, _lib.MAX_CONDITIONS))
        if a.replicas is not None and len(a.replicas) != K:
            raise ValueError("dpm_solver_b200: a multi-condition step takes one replica per condition")
        n, mdt = ref.numel(), a.e_cond.dtype
        maps = None if a.masks is None else self._cond_maps(a, ref, layout, keep)
        ecs = [self._check(e, "e_conds[%d]" % k, ref.device, n, mdt, layout) for k, e in enumerate(a.e_conds)]
        keep.extend(ecs)
        reps = None
        if a.replicas is not None and a.form != FORM_NONE:
            for k, r in enumerate(a.replicas):
                self._check(r, "replicas[%d]" % k, ref.device, n, sdt)
                if self._layout(r) != layout:
                    raise ValueError("dpm_solver_b200: replicas must be dense and laid out like out")
            reps = (C.c_void_p * K)(*[r.data_ptr() for r in a.replicas])
        d.out2 = None
        ecp, sc = (C.c_void_p * K)(*[e.data_ptr() for e in ecs]), (C.c_float * K)(*a.scales)
        if maps is None:
            self._launch(ref.device, self._lib.dpm_step_multi, C.byref(d), ecp, sc, C.c_int(K), reps)
        else:
            self._launch(ref.device, self._lib.dpm_step_multi_masked, C.byref(d), ecp, sc, maps, C.c_int(K), reps)

    @staticmethod
    def _cond_maps(a: StepArgs, ref, layout, keep):
        """The dpm_cond_map array of `a.masks`, each map checked against the launch's size and per_sample."""
        n = ref.numel()
        if a.per_sample <= 0 or n % a.per_sample:
            raise ValueError("dpm_solver_b200: a masked multi-condition step needs per_sample dividing numel")
        maps = (_lib.CondMap * len(a.masks))()
        for k, m in enumerate(a.masks):
            if m is None:
                continue
            w, period, stride = m if isinstance(m, tuple) else m.weights(tuple(ref.shape), layout, ref.device)
            if not w.is_cuda or w.device != ref.device or w.dtype != torch.float32 or not w.is_contiguous():
                raise TypeError("dpm_solver_b200: a weight map must be a contiguous fp32 tensor on the tensors' device")
            if period <= 0 or a.per_sample % period or stride not in (0, period) \
                    or w.numel() != (period if stride == 0 else period * (n // a.per_sample)):
                raise ValueError("dpm_solver_b200: weight map {} does not fit period {} and sample stride {}".format(
                    k, period, stride))
            keep.append(w)
            maps[k].w, maps[k].period, maps[k].sample_stride = w.data_ptr(), period, stride
        return maps

    def _step_sde(self, a: StepArgs, d, ref, layout, keep) -> None:
        """dpm_step_sde: the update of `a` plus a.sde.cz times its noise (d already filled). The noise is drawn inside the
        launch from the generator's (seed, offset), the generator advanced as normal_ would advance it; under CUDA-graph
        capture, or when the launch's layout is not x's own, it is drawn by torch instead (graph-safe) and read."""
        if a.form not in (FORM_LIN1, FORM_DIFF2, FORM_MS3) or a.c0_on_old or a.raw_round or a.coef_dev is not None \
                or a.e_conds is not None or a.apg_words is not None or a.cfgpp_g is not None:
            raise ValueError("dpm_solver_b200: an SDE step is a multistep LIN1 / DIFF2 / MS3 update with one scalar or "
                             "per-sample scale, rescale, CFG-Zero* or TCFG words")
        gen = a.sde.generator
        if gen is not None and not same_device(gen.device, ref.device):
            raise ValueError("dpm_solver_b200: the generator is on {}, x on {}".format(gen.device, ref.device))
        s = _lib.SdeDesc()
        s.cz = a.sde.cz
        if torch.cuda.is_current_stream_capturing() or self._layout(a.x) != layout:
            z = torch.empty_like(a.x, dtype=torch.float32).normal_(generator=gen)
            z = self._check(z, "z", ref.device, ref.numel(), torch.float32, layout)
            keep.append(z)
            s.z = z.data_ptr()
        else:
            with torch.cuda.device(ref.device):
                s.seed, s.offset = self._philox_state(ref.device, ref.numel(), self._lib, gen)
        for name, v in (("guidance", a.guidance_b), ("ratio", a.ratio), ("s_star", a.cfgzero_s),
                        ("tcfg_words", a.tcfg_w)):
            if v is not None:
                setattr(s, name, v.data_ptr())
        s.phi, s.one_minus_phi = a.phi, 1.0 - a.phi
        self._launch(ref.device, self._lib.dpm_step_sde, C.byref(d), C.byref(s))

    def _step_unipc(self, a: StepArgs, d, ref, sdt, layout, keep) -> None:
        """dpm_step_unipc: the UniPC words, m_{i-3} and the corrected-state output of a launch (d already filled)."""
        if a.e_conds is not None or a.guidance_b is not None or a.ratio is not None or a.apg_words is not None \
                or a.cfgzero_s is not None or a.cfgpp_g is not None or a.tcfg_w is not None:
            raise ValueError("dpm_solver_b200: a UniPC step takes one guidance scale, without rescale, APG, CFG-Zero*, "
                             "CFG++ or TCFG")
        w, u = a.unipc, _lib.UniDesc()
        n = ref.numel()
        if a.m3 is not None:
            m3 = self._check(a.m3, "m3", ref.device, n, sdt, layout)
            keep.append(m3)
            u.m3 = m3.data_ptr()
        if a.out_c is not None:
            self._check(a.out_c, "out_c", ref.device, n, sdt)
            if self._layout(a.out_c) != layout:
                raise ValueError("dpm_solver_b200: out_c must be dense and laid out like the inputs")
            u.out_c = a.out_c.data_ptr()
        u.pc, u.pp = int(w.pc), int(w.pp)
        u.cd[0], u.cd[1] = w.cd
        u.ct, u.a, u.c0 = w.ct, w.a, w.c0
        u.cp[0], u.cp[1] = w.cp
        self._launch(ref.device, self._lib.dpm_step_unipc, C.byref(d), C.byref(u))

    def replicate(self, x: torch.Tensor, copies: int) -> torch.Tensor:
        """torch.cat([x] * copies) -- one read, `copies` writes (dpm_replicate); layout of x kept."""
        if x.dtype not in _DTYPE_CODE:
            raise TypeError(f"dpm_solver_b200: unsupported dtype {x.dtype} for replicate")
        layout = self._layout(x)
        if layout is None:
            x, layout = x.contiguous(), "c"
        shape = (copies * x.shape[0],) + tuple(x.shape[1:])
        if layout == "cl":
            out = torch.empty(shape, dtype=x.dtype, device=x.device,
                              memory_format=torch.channels_last if x.dim() == 4 else torch.channels_last_3d)
        else:
            out = torch.empty(shape, dtype=x.dtype, device=x.device)
        self._check(x, "x", x.device, x.numel(), layout=layout)
        self._launch(x.device, self._lib.dpm_replicate, C.c_void_p(out.data_ptr()), C.c_void_p(x.data_ptr()),
                     C.c_uint64(x.numel()), C.c_int(copies), C.c_int(_DTYPE_CODE[x.dtype]))
        return out

    def cfg_rescale_ratio(self, e_cond: torch.Tensor, e_uncond: torch.Tensor, guidance) -> torch.Tensor:
        """Per-sample r = std(e_cond_b) / std(g_b), g = e_uncond + guidance*(e_cond - e_uncond), as fp32 [B] on the
        device (dpm_cfg_rescale_ratio). Both halves keep a shared dense layout: a sample is one contiguous block
        in row-major and in channels_last storage alike. `guidance` may be a contiguous fp32 device tensor of B
        per-sample scales (dpm_cfg_rescale_ratio_guided)."""
        blocks = [("e_cond", e_cond), ("e_uncond", e_uncond)]
        if not torch.is_tensor(guidance):
            return self._words(self._lib.dpm_cfg_rescale_ratio, self._lib.dpm_cfg_rescale_workspace, (), blocks,
                               lambda p, ps, n, dt: (*p, C.c_float(guidance), ps, n, dt))

        def guided_args(p, ps, n, dt):
            # (checked once _words has checked the halves, so that a bad half is reported first)
            if not guidance.is_cuda or guidance.dtype != torch.float32 or not guidance.is_contiguous() \
                    or guidance.device != e_cond.device or guidance.numel() != e_cond.shape[0]:
                raise ValueError("dpm_solver_b200: per-sample guidance must be a contiguous fp32 [B] tensor on the "
                                 "tensors' device")
            return (*p, C.c_void_p(guidance.data_ptr()), ps, n, dt)
        return self._words(self._lib.dpm_cfg_rescale_ratio_guided, self._lib.dpm_cfg_rescale_workspace, (), blocks,
                           guided_args)

    def _launch(self, device, fn, *args):
        """Call a C-ABI entry on torch's current stream of `device` (device guard only if needed)."""
        idx = device.index
        if torch.cuda.current_device() == idx:
            rc = fn(*args, C.c_void_p(_raw_stream(idx)))
        else:
            with torch.cuda.device(device):
                rc = fn(*args, C.c_void_p(_raw_stream(idx)))
        if rc != 0:
            _lib.check(rc)

    def dynamic_threshold(self, a: StepArgs, q: float, max_val: float, return_stats: bool = False):
        """Per-sample s_b = max(quantile(|x0_b|, q), max_val) -> fp32 [B].
        return_stats=True also returns the pipeline's per-sample header words (int32 [B, 8]:
        lo key, hi key, #below, #inside, path (1 bracket / 2 exact fallback), ...) for diagnostics."""
        if a.guidance_b is not None or a.e_conds is not None or a.apg_words is not None or a.cfgzero_s is not None \
                or a.tcfg_w is not None:
            raise ValueError("dpm_solver_b200: the quantile takes one guidance scale; materialise a per-sample, "
                             "multi-condition, APG, CFG-Zero* or TCFG combine first")
        d, keep, ref, _, _ = self._fill(a)
        if a.per_sample <= 0 or ref.numel() % a.per_sample:
            raise ValueError("dpm_solver_b200: per_sample must divide numel")
        nb = ref.numel() // a.per_sample
        s = torch.empty(nb, dtype=torch.float32, device=ref.device)
        ws_bytes = int(self._lib.dpm_dynamic_threshold_workspace(nb, a.per_sample))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=ref.device) if ws_bytes else None
        self._launch(ref.device, self._lib.dpm_dynamic_threshold, C.c_void_p(s.data_ptr()), C.byref(d),
                     C.c_float(q), C.c_float(max_val), C.c_void_p(ws.data_ptr() if ws is not None else None),
                     C.c_size_t(ws_bytes))
        if return_stats:
            hdr = ws[:nb * 32].view(torch.int32).reshape(nb, 8).clone() if ws is not None else None
            return s, hdr
        return s

    def error_norm(self, x_higher, x_lower, x_prev, atol: float, rtol: float, out=None) -> torch.Tensor:
        """E of dpm_solver_adaptive (:999-1001) as a device fp32 tensor of shape (1,)."""
        n, dev = x_higher.numel(), x_higher.device
        ts = [self._check(t, w, dev, n, x_higher.dtype) for t, w in ((x_higher, "x_higher"), (x_lower, "x_lower"), (x_prev, "x_prev"))]
        per_sample = n // x_higher.shape[0]
        if out is None:
            out = torch.empty(1, dtype=torch.float32, device=dev)
        ws_bytes = int(self._lib.dpm_adaptive_error_workspace(n, per_sample))
        ws = torch.empty(max(ws_bytes, 4), dtype=torch.uint8, device=dev)
        self._launch(dev, self._lib.dpm_adaptive_error, C.c_void_p(out.data_ptr()), C.c_void_p(ts[0].data_ptr()),
                     C.c_void_p(ts[1].data_ptr()), C.c_void_p(ts[2].data_ptr()), C.c_float(atol), C.c_float(rtol),
                     C.c_uint64(per_sample), C.c_uint64(n), C.c_int(_DTYPE_CODE[x_higher.dtype]),
                     C.c_void_p(ws.data_ptr()), C.c_size_t(ws_bytes))
        return out

    def duplicate(self, x: torch.Tensor) -> torch.Tensor:
        """torch.cat([x] * 2) (model_wrapper :326) -- one read, two bulk writes; layout of x kept."""
        if x.dtype not in _DTYPE_CODE:
            return torch.cat([x] * 2)
        layout = self._layout(x)
        if layout is None:
            x, layout = x.contiguous(), "c"
        shape = (2 * x.shape[0],) + tuple(x.shape[1:])
        if layout == "cl":
            out = torch.empty(shape, dtype=x.dtype, device=x.device,
                              memory_format=torch.channels_last if x.dim() == 4 else torch.channels_last_3d)
        else:
            out = torch.empty(shape, dtype=x.dtype, device=x.device)
        self._check(x, "x", x.device, x.numel(), layout=layout)
        self._launch(x.device, self._lib.dpm_duplicate, C.c_void_p(out.data_ptr()), C.c_void_p(x.data_ptr()),
                     C.c_uint64(x.numel()), C.c_int(_DTYPE_CODE[x.dtype]))
        return out

    def adaptive_controller(self, ns, device, **kw) -> "AdaptiveController":
        """Device-resident step-size controller of dpm_solver_adaptive (csrc/adaptive_ctl.cu)."""
        return AdaptiveController(self, ns, device, **kw)

    # -- noise drawn inside the kernel (torch.randn-compatible Philox; csrc/philox.cu) ----------------------
    @staticmethod
    def _philox_state(device, numel: int, lib, generator=None):
        """(seed, offset) of the torch CUDA generator for a randn of `numel` elements, advancing it exactly as
        ATen's normal_ kernel would (so later torch RNG calls see the state they would have seen)."""
        gen = generator if generator is not None else torch.cuda.default_generators[device.index]
        grid, inc = C.c_uint32(0), C.c_uint64(0)
        _lib.check(lib.dpm_philox_policy(C.c_uint64(numel), C.byref(grid), C.byref(inc)))
        seed, offset = gen.initial_seed(), gen.get_offset()
        gen.set_offset(offset + inc.value)
        return seed, offset

    def add_noise_philox(self, x: torch.Tensor, alphas, sigmas, out_dtype, generator=None) -> torch.Tensor:
        """[T, *x.shape] = alpha_i * x + sigma_i * randn, the noise generated in registers (reference :1023-1026)."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("dpm_solver_b200: in-kernel noise reads the generator state on the host; pass `noise=` under CUDA-graph capture")
        x = self._check(x, "x", x.device, x.numel())
        T = len(alphas)
        out = torch.empty((T,) + tuple(x.shape), dtype=out_dtype, device=x.device)
        with torch.cuda.device(x.device):
            seed, offset = self._philox_state(x.device, T * x.numel(), self._lib, generator)
        fa = (C.c_float * T)(*alphas)
        fs = (C.c_float * T)(*sigmas)
        self._launch(x.device, self._lib.dpm_add_noise_philox, C.c_void_p(out.data_ptr()), C.c_void_p(x.data_ptr()),
                     C.c_uint64(x.numel()), C.c_int(T), fa, fs, C.c_uint64(seed), C.c_uint64(offset),
                     C.c_int(_DTYPE_CODE[x.dtype]), C.c_int(_DTYPE_CODE[out_dtype]))
        return out

    def diffedit_corrector(self, x, x0, mask, alpha: float, sigma: float, generator=None) -> torch.Tensor:
        """x*mask + (1 - mask)*(alpha*x0 + sigma*randn_like(x0)) in one launch (diffedit_inpaint.ipynb corrector_fn)."""
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("dpm_solver_b200: in-kernel noise reads the generator state on the host; not capturable")
        n = x.numel()
        x = self._check(x, "x", x.device, n)
        x0 = self._check(x0, "x0", x.device, n, x.dtype)
        if mask.dtype != torch.float32 or not mask.is_contiguous() or n % max(mask.numel(), 1) \
                or tuple(mask.shape) != tuple(x.shape[x.dim() - mask.dim():]):
            mask = mask.to(torch.float32).expand(x.shape).contiguous()        # any other broadcast: materialise
        if mask.device != x.device:
            raise RuntimeError("dpm_solver_b200: `mask` must live on the device of x")
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            seed, offset = self._philox_state(x.device, n, self._lib, generator)
        self._launch(x.device, self._lib.dpm_diffedit_corrector, C.c_void_p(out.data_ptr()), C.c_void_p(x.data_ptr()),
                     C.c_void_p(x0.data_ptr()), C.c_void_p(mask.data_ptr()), C.c_uint64(mask.numel()), C.c_uint64(n),
                     C.c_float(alpha), C.c_float(sigma), C.c_uint64(seed), C.c_uint64(offset), C.c_int(_DTYPE_CODE[x.dtype]))
        return out

    def prepare(self, a: StepArgs) -> Optional["PreparedStep"]:
        """Freeze the descriptor of a launch whose scalars will not change (one step of a cached coefficient plan):
        later launches of the same step only patch the tensor pointers. None if the launch is not eligible."""
        return PreparedStep.build(self, a)

    def launch_count(self) -> int:
        return int(self._lib.dpm_launch_count())

    def set_tuning(self, variant: int = 2, threads: int = 0, ctas_per_sm: int = 0) -> None:
        _lib.check(self._lib.dpm_set_tuning(variant, threads, ctas_per_sm))


class AdaptiveController:
    """State, coefficient blocks and time labels of dpm_solver_adaptive (:956-1010) in device memory, plus the three
    tiny kernels that advance them (dpm_adaptive_init / _plan / _decide) and the conditional commit
    (dpm_select_copy). `read()` is the only host synchronisation."""

    SUPPORTED = ("discrete", "linear", "flow")

    def __init__(self, be: "CudaBackend", ns, device, order: int, predict_x0: bool, taylor: bool, t_0: float,
                 theta: float, t_err: float, discrete_input: bool):
        if ns.schedule not in self.SUPPORTED:
            raise ValueError("the device controller supports the 'discrete', 'linear' and 'flow' schedules")
        self.be, self.dev = be, torch.device(device)
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.state = torch.zeros(16, **f32)
        self.coef = torch.zeros(4, 16, **f32)
        self.times = torch.zeros(6, **f32)
        self.E = torch.zeros(1, **f32)
        c = self.ctl = _lib.AdaptiveCtl()
        self._keep = []
        if ns.schedule == "discrete":
            tabs = ns._table(self.dev)[:4]
            self._keep = [t.to(torch.float32).contiguous() for t in tabs]
            c.schedule_kind, c.table_len = 0, self._keep[0].numel()
            c.t_array, c.log_alpha_array, c.log_alpha_flipped, c.t_flipped = (t.data_ptr() for t in self._keep)
            c.inv_total_N = 1. / ns.total_N
        elif ns.schedule == "flow":
            c.schedule_kind, c.table_len = 2, 0
            # shift - 1 in double, each scalar rounded to fp32 once, as torch rounds the python-float operands
            c.flow_shift, c.flow_shift_minus_1, c.flow_time_scale = ns.shift, ns.shift - 1., ns.time_scale
            c.inv_total_N = 1. / ns.total_N
        else:
            c.schedule_kind, c.table_len = 1, 0
            c.beta_0, c.beta_1_minus_beta_0 = ns.beta_0, ns.beta_1 - ns.beta_0
            c.beta_0_sq = ns.beta_0 ** 2          # squared in double, rounded once (inverse_lambda :162)
            c.inv_total_N = 1. / ns.total_N
        c.discrete_time_input = int(bool(discrete_input))
        c.order, c.predict_x0, c.taylor = order, int(bool(predict_x0)), int(bool(taylor))
        c.t_0, c.theta, c.t_err = t_0, theta, t_err
        c.state, c.coef, c.times, c.error = (t.data_ptr() for t in (self.state, self.coef, self.times, self.E))
        self._ref = C.byref(c)

    def init(self, t_T: float, h_init: float) -> None:
        self.be._launch(self.dev, self.be._lib.dpm_adaptive_init, self._ref, C.c_float(t_T), C.c_float(h_init))

    def plan(self) -> None:
        self.be._launch(self.dev, self.be._lib.dpm_adaptive_plan, self._ref)

    def decide(self) -> None:
        self.be._launch(self.dev, self.be._lib.dpm_adaptive_decide, self._ref)

    def select_copy(self, dst: torch.Tensor, src: torch.Tensor) -> None:
        """dst <- src iff the last decide() accepted the step."""
        if dst.shape != src.shape or dst.dtype != src.dtype or CudaBackend._layout(dst) is None:
            raise ValueError("select_copy: tensors of one shape and dtype, the destination dense")
        if src.stride() != dst.stride():
            # (a channels_last network under a row-major x_T, or the reverse: the byte copy below needs dst's order)
            src = torch.empty_like(dst).copy_(src)
        self.be._launch(self.dev, self.be._lib.dpm_select_copy, C.c_void_p(dst.data_ptr()), C.c_void_p(src.data_ptr()),
                        C.c_void_p(self.state.data_ptr()), C.c_uint64(dst.numel() * dst.element_size()))

    def block(self, i: int) -> torch.Tensor:
        return self.coef[i]

    def time(self, j: int) -> torch.Tensor:
        return self.times[j:j + 1]

    def input_time(self, j: int) -> torch.Tensor:
        return self.times[3 + j:4 + j]

    def read(self):
        """(done, nfe, iterations): the one device->host read of a chunk."""
        st = self.state.cpu().view(torch.int32)
        return int(st[6]), int(st[5]), int(st[8])


class PreparedStep:
    """One step of a cached coefficient plan, ready to launch: a filled `dpm_step_desc` whose scalar fields are final.
    `launch()` validates the tensors of this call with a handful of attribute reads (dtype, size, density, device),
    patches the pointers, allocates the outputs and calls the C-ABI -- the per-step host path of a steady-state
    sample() loop (tools/host_overhead.py). Anything unusual (other layout, dtype, device, size) returns None and the
    caller takes the general path (`CudaBackend.step`)."""

    __slots__ = ("be", "d", "ref_d", "fn", "n", "dev", "dev_index", "sdt", "mdt", "shape", "shape2", "need_out",
                 "need_m", "fields", "dup", "ptrs", "esize")

    ORDER = ("x", "xe", "m0", "m1", "m2", "e_cond", "e_uncond")     # launch() takes its tensors in this order
    # index of every pointer field inside struct dpm_step_desc (its first 11 members are pointers)
    _PTR = {"x": 0, "xe": 1, "m0": 2, "m1": 3, "m2": 4, "m_out": 5, "out": 6, "out2": 7, "e_cond": 8, "e_uncond": 9}

    @staticmethod
    def build(be: "CudaBackend", a: StepArgs) -> Optional["PreparedStep"]:
        if a.thr is not None or a.raw_round or a.ratio is not None or a.guidance_b is not None \
                or a.e_conds is not None or a.coef_dev is not None or a.unipc is not None \
                or a.apg_words is not None or a.cfgzero_s is not None or a.cfgpp_g is not None \
                or a.tcfg_w is not None or a.sde is not None or a.out is not None and a.out2 is None:
            # (a rescaled step reads a fresh ratio tensor every evaluation, an APG one fresh words, a CFG-Zero* one fresh
            # scales s*, a TCFG one fresh words (wu, wc), a CFG++ one goes through its own entry point, a guided one a
            # scales tensor the descriptor does not carry, a multi-condition one K outputs and scales it does not
            # carry, one with device coefficients a block the descriptor would point into without owning it: never
            # frozen)
            return None
        ref = a.reference_tensor()
        if not ref.is_contiguous():
            return None
        for t in a.state_tensors() + a.model_tensors():
            if not t.is_contiguous() or t.device != ref.device:
                return None
        d, keep, ref, sdt, layout = be._fill(a)
        if layout != "c":
            return None
        self = PreparedStep()
        self.be, self.d, self.ref_d, self.fn = be, d, C.byref(d), be._lib.dpm_step
        self.n, self.dev, self.dev_index = ref.numel(), ref.device, ref.device.index
        self.sdt = sdt
        self.mdt = a.e_cond.dtype if a.e_cond is not None else sdt
        self.shape = tuple(ref.shape)
        self.shape2 = (2 * self.shape[0],) + self.shape[1:]
        self.esize = torch.empty((), dtype=sdt).element_size()
        # the descriptor's pointer members as a uint64 array: patching one is a numpy scalar store, not a ctypes setattr
        import numpy as np
        self.ptrs = np.frombuffer((C.c_char * C.sizeof(d)).from_buffer(d), dtype=np.uint64, count=11)
        self.need_out = a.form != FORM_NONE
        self.need_m = a.n_model > 0 and (a.want_m_out or a.form == FORM_NONE)
        self.dup = a.out2 is not None
        # (descriptor field, StepArgs attribute, expected dtype) of every input tensor this launch reads
        # (pointer slot, position in launch()'s tensor tuple, expected dtype) of every input this launch reads
        self.fields = tuple((self._PTR[name], pos, self.mdt if name in ("e_cond", "e_uncond") else sdt)
                            for pos, name in enumerate(self.ORDER) if getattr(a, name) is not None)
        return self

    def launch(self, tensors: tuple):
        """tensors: (x, xe, m0, m1, m2, e_cond, e_uncond) (`ORDER`; entries the frozen launch does not read are
        ignored). Returns (m_out, out, x_in) -- x_in is the doubled CFG batch when the step was prepared with a second
        output copy -- or None when a tensor does not look like the ones the step was prepared for."""
        n, dev, idx, ptrs = self.n, self.dev, self.dev_index, self.ptrs
        for f, pos, dt in self.fields:
            t = tensors[pos]
            if t is None or t.dtype is not dt or t.numel() != n or not t.is_contiguous() or t.get_device() != idx:
                return None
            ptrs[f] = t.data_ptr()
        m_out = out = x_in = None
        if self.need_m:
            m_out = torch.empty(self.shape, dtype=self.sdt, device=dev)
            ptrs[5] = m_out.data_ptr()
        if self.need_out:
            if self.dup:
                x_in = torch.empty(self.shape2, dtype=self.sdt, device=dev)
                out = x_in[:self.shape[0]]
                base = x_in.data_ptr()
                ptrs[6] = base
                ptrs[7] = base + n * self.esize
            else:
                out = torch.empty(self.shape, dtype=self.sdt, device=dev)
                ptrs[6] = out.data_ptr()
        if torch.cuda.current_device() == idx:
            rc = self.fn(self.ref_d, _raw_stream(idx))
        else:
            with torch.cuda.device(dev):
                rc = self.fn(self.ref_d, _raw_stream(idx))
        if rc != 0:
            _lib.check(rc)
        return m_out, out, x_in


_backend = None


def backend():
    """The active executor (CudaBackend unless a test installed another one)."""
    global _backend
    if _backend is None:
        _backend = CudaBackend()
    return _backend


def set_backend(b) -> None:
    """Install an executor with the CudaBackend interface. Used by tests/ only."""
    global _backend
    _backend = b


# ---- convenience wrappers, named after the reference functions they replace -----------------

def lincomb(x, ms, a, cs, out=None):
    """out = a*x + sum_j cs[j]*ms[j], 1 <= len(ms) <= 3, unfused fp32 chain, left to right."""
    k = len(ms)
    if not 1 <= k <= 3 or len(cs) != k:
        raise ValueError("lincomb takes 1..3 (tensor, coefficient) pairs")
    a_ = StepArgs(form=(FORM_LIN1, FORM_LIN2, FORM_LIN3)[k - 1], x=x, m0=ms[0],
                  m1=ms[1] if k > 1 else None, m2=ms[2] if k > 2 else None, a=a, c0=cs[0],
                  c1=cs[1] if k > 1 else 0.0, c2=cs[2] if k > 2 else 0.0, out=out)
    return backend().step(a_)[1]


def cfg_combine(eps_uncond, eps_cond, scale):
    """model_wrapper.model_fn :329-330."""
    a_ = StepArgs(form=FORM_NONE, n_model=2, e_cond=eps_cond, e_uncond=eps_uncond, guidance=scale,
                  state_dtype=eps_cond.dtype)
    return backend().step(a_)[0]


__all__ = ["StepArgs", "CudaBackend", "backend", "set_backend", "lincomb", "cfg_combine",
           "SdeNoise", "SUPPORTED_DTYPES", "FORM_NONE", "FORM_LIN1", "FORM_LIN2", "FORM_LIN3", "FORM_DIFF2",
           "FORM_MS3", "FORM_SS3T"]
