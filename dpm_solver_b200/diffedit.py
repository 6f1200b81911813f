"""Fused DiffEdit corrector (SURVEY 8f-3): a `correcting_xt_fn` for `DPM_Solver` / `DPMSolverSampler.sample`.

The reference's inpainting example (examples/stable-diffusion/scripts/diffedit_inpaint.ipynb, `corrector_fn`)
re-noises the encoded source image at every solver step and blends it in outside the edit mask:

    def corrector_fn(x, t, step):
        ratio = sampler.time_to_ratio(t)
        stochastic_intermediate = sampler.stochastic_encode(init_latent, ratio)   # alpha*x0 + sigma*randn (sampler.py:92-96)
        return x * mask + (1 - mask) * stochastic_intermediate

-- a randn, the three ops of add_noise and four blend ops, eight full-tensor passes. `DiffEditCorrector` is the
same function as ONE kernel (csrc/philox.cu): the noise is drawn in registers by the generator torch.randn uses,
so for fp32 latents and the same generator state the result is bit-identical to the expression above. (16-bit
latents: the same fp32 arithmetic, rounded to the latents' type once on store; the reference's expression promotes
to fp32 and returns fp32.)
"""
from __future__ import annotations

import torch

from . import ops

__all__ = ["DiffEditCorrector"]


class DiffEditCorrector:
    """`DiffEditCorrector(noise_schedule, init_latent, mask, time_fn)(x, t, step)`.

    time_fn maps the solver's current time `t` (a tensor) to the time whose noise level the source image is
    re-noised to -- the notebook's `lambda t: sampler.ratio_to_time(sampler.time_to_ratio(t))`; default: `t` itself.
    The (alpha, sigma) of a time label are cached under the label's identity (its memory, version and device, and
    the `time_fn` in use), never under the step number: a solver hands over the same cached label tensors on every
    run of a configuration, so steady-state calls read nothing back from the device, while another `steps`, `t_end`,
    `skip_type`, `method` or `time_fn` -- which map step k to another time -- meet other labels and are recomputed.
    `generator`, when given, must be a generator of x's device (ValueError otherwise)."""

    _CACHE_MAX = 1024

    def __init__(self, noise_schedule, init_latent, mask, time_fn=None, generator=None):
        self.noise_schedule = noise_schedule
        self.init_latent = init_latent
        self.mask = mask.to(torch.float32).contiguous()
        self.time_fn = time_fn
        self.generator = generator
        self._scalars = {}

    def _alpha_sigma(self, t, step=None):
        """(alpha, sigma, time) the source is re-noised to at label `t`; `step` does not enter."""
        t = torch.as_tensor(t)
        key = (t.data_ptr(), t._version, t.device, id(self.time_fn))
        hit = self._scalars.get(key)
        if hit is None:
            te = t if self.time_fn is None else self.time_fn(t)
            te = torch.as_tensor(te, dtype=torch.float32).reshape(-1)[:1].cpu()      # one read-back per distinct label
            # stochastic_encode rebuilds the label in the latent's dtype (sampler.py:94) before add_noise
            te = te.to(self.init_latent.dtype).to(torch.float32) if self.init_latent.dtype != torch.float32 else te
            ns = self.noise_schedule
            # the label and the time_fn are kept next to the scalars so that neither the memory nor the id in the key
            # can be recycled while the entry lives
            hit = (float(ns.marginal_alpha(te)), float(ns.marginal_std(te)), float(te), t, self.time_fn)
            if len(self._scalars) >= self._CACHE_MAX:
                self._scalars.clear()
            self._scalars[key] = hit
        return hit[:3]

    def __call__(self, x, t, step):
        g = self.generator
        if g is not None and (g.device.type != x.device.type or g.device.index not in (None, x.device.index)):
            raise ValueError("DiffEditCorrector: `generator` is on {}, x on {}".format(g.device, x.device))
        alpha, sigma, _ = self._alpha_sigma(t, step)
        be = ops.backend()
        x0 = self.init_latent
        if x0.dtype != x.dtype:
            x0 = x0.to(x.dtype)
        return be.diffedit_corrector(x, x0.expand(x.shape) if x0.shape != x.shape else x0, self.mask.to(x.device),
                                     alpha, sigma, self.generator)
