"""Oracle of regional guidance (model_wrapper's guidance_mask) -- TEST INFRASTRUCTURE.

`MaskOracle`: the numpy executor (cfgpp_oracle.CFGPPOracle: every parameterisation, guidance form and solver launch)
plus dpm_step_multi_masked as include/dpm_solver_b200.h states it. The weight of condition k at element i (storage
order) is maps[k].w[b*sample_stride + (i - b*per_sample) % period]; w_k = fl32(s_k)*m_k(i) is formed once, rounded to
fp32, and the executor's own multi-condition combine then runs with that per-element array in place of s_k, so every
parameterisation converts each block exactly as without masks.
"""
import dataclasses

import numpy as np
import torch

from cfgpp_oracle import CFGPPOracle
from oracle_backend import _np

f32 = np.float32


def _layout(t):
    if t.is_contiguous():
        return "c"
    if t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last):
        return "cl"
    if t.dim() == 5 and t.is_contiguous(memory_format=torch.channels_last_3d):
        return "cl"
    return "c"


def weight_array(m, shape, layout, per_sample):
    """The logical-shape fp32 array m_k(i) of one map entry (None: ones) for a launch over `shape` in `layout`."""
    n = int(np.prod(shape))
    if m is None:
        return np.ones(shape, f32)
    w, period, stride = m
    wf = _np(w).reshape(-1)
    i = np.arange(n, dtype=np.int64)
    b = i // per_sample
    flat = wf[b * stride + (i - b * per_sample) % period].astype(f32)     # storage order
    if layout == "cl":
        d = len(shape)
        st = (shape[0],) + tuple(shape[2:]) + (shape[1],)
        return np.ascontiguousarray(flat.reshape(st).transpose(0, d - 1, *range(1, d - 1)))
    return flat.reshape(shape)


class MaskOracle(CFGPPOracle):
    """The numpy executor with dpm_step_multi_masked (StepArgs.masks)."""

    def step(self, a):
        if getattr(a, "masks", None) is not None:
            self.log.append(("masked", a.form))
        return super().step(a)

    def _model_value(self, a, thr=None):
        if getattr(a, "masks", None) is None or a.e_conds is None:
            return super()._model_value(a, thr)
        ref = a.reference_tensor()
        shape, layout = tuple(ref.shape), _layout(ref)
        assert a.per_sample > 0 and ref.numel() % a.per_sample == 0
        ws = []
        for s, m in zip(a.scales, a.masks):
            if m is not None and not isinstance(m, tuple):
                m = m.weights(shape, layout, ref.device)
            with np.errstate(all="ignore"):
                ws.append(f32(s) if m is None else (f32(s) * weight_array(m, shape, layout, a.per_sample)).astype(f32))
        return super()._model_value(dataclasses.replace(a, scales=tuple(ws), masks=None), thr)
