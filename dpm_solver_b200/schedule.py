"""Noise schedule scalars: log(alpha_t), alpha_t, sigma_t, lambda_t and lambda^-1, for the reference's VP schedules
(`NoiseScheduleVP`), for flow-matching models on the linear path (`NoiseScheduleFlow`) and for EDM-preconditioned
models (`NoiseScheduleEDM`).

API-compatible with `NoiseScheduleVP` of the reference (dpm_solver_pytorch.py:6-167) -- same
constructor, attributes and methods -- but every method is a handful of vectorised ops: the
reference's `interpolate_fn` (cat + sort + argmin + 3 where + 4 gather on a [N,1,K+1] tensor,
:1253-1292) becomes one `searchsorted` + four gathers. The arithmetic keeps the reference's fp32
operation order (`y0 + (x - x0) * (y1 - y0) / (x1 - x0)`, :1291), so results are bit-identical;
the solver evaluates these on HOST tensors once per run (see plan.py), never per step on device.
"""
from __future__ import annotations

import torch

__all__ = ["NoiseScheduleVP", "NoiseScheduleFlow", "NoiseScheduleEDM", "interpolate_fn", "expand_dims"]


def _piecewise_linear(x: torch.Tensor, xp: torch.Tensor, yp: torch.Tensor) -> torch.Tensor:
    """y(x) for ascending keypoints xp/yp (1-D), linear extrapolation outside (reference :1253).

    The reference finds the bracket by sorting [x, xp...] (x first, so on ties x precedes the
    equal keypoint): with i = #{xp < x} the bracket is [xp[i-1], xp[i]], clamped to the first /
    last interval. searchsorted(right=False) returns exactly that i.
    """
    K = xp.shape[0]
    i = torch.searchsorted(xp, x.contiguous(), right=False)
    j0 = (i - 1).clamp_(0, K - 2)
    x0, x1 = xp[j0], xp[j0 + 1]
    y0, y1 = yp[j0], yp[j0 + 1]
    return y0 + (x - x0) * (y1 - y0) / (x1 - x0)


def interpolate_fn(x: torch.Tensor, xp: torch.Tensor, yp: torch.Tensor) -> torch.Tensor:
    """Drop-in for the reference utility (:1253-1292): x [N,C], xp/yp [C,K] -> [N,C]."""
    cols = [_piecewise_linear(x[:, c], xp[c], yp[c]) for c in range(xp.shape[0])]
    return torch.stack(cols, dim=1)


def expand_dims(v: torch.Tensor, dims: int) -> torch.Tensor:
    """[N] -> [N,1,...,1] with `dims` dimensions (reference :1295-1305)."""
    return v[(...,) + (None,) * (dims - 1)]


class NoiseScheduleVP:
    """Forward VP SDE wrapper; see the reference docstring (:16-92) for the maths.

    schedule='discrete': piecewise-linear log(alpha) over t_i = (i+1)/N from `betas` or
    `alphas_cumprod` (tail clipped where lambda < -5.1, :114-125); schedule='linear': the
    continuous VPSDE with beta_0, beta_1 (:134); schedule='cosine' is accepted for the older
    vendored copies of the solver (examples/stable-diffusion/.../dpm_solver.py:114-175).
    """

    def __init__(self, schedule="discrete", betas=None, alphas_cumprod=None, continuous_beta_0=0.1,
                 continuous_beta_1=20., dtype=torch.float32):
        if schedule not in ["discrete", "linear", "cosine"]:
            raise ValueError("Unsupported noise schedule {}. The schedule needs to be 'discrete' or "
                             "'linear'".format(schedule))
        self.schedule = schedule
        self.T = 1.
        self._tables = {}
        if schedule == "discrete":
            if betas is not None:
                log_alphas = 0.5 * torch.log(1 - betas).cumsum(dim=0)
            else:
                assert alphas_cumprod is not None
                log_alphas = 0.5 * torch.log(alphas_cumprod)
            log_alphas = self.numerical_clip_alpha(log_alphas)
            self.log_alpha_array = log_alphas.reshape((1, -1,)).to(dtype=dtype)
            self.total_N = self.log_alpha_array.shape[1]
            self.t_array = torch.linspace(0., 1., self.total_N + 1)[1:].reshape((1, -1)).to(dtype=dtype)
        else:
            self.total_N = 1000
            self.beta_0 = continuous_beta_0
            self.beta_1 = continuous_beta_1
            if schedule == "cosine":
                import math
                self.cosine_s = 0.008
                self.cosine_beta_max = 999.
                self.cosine_t_max = math.atan(self.cosine_beta_max * (1. + self.cosine_s) / math.pi) * 2. \
                    * (1. + self.cosine_s) / math.pi - self.cosine_s
                self.cosine_log_alpha_0 = math.log(math.cos(self.cosine_s / (1. + self.cosine_s) * math.pi / 2.))
                self.T = 0.9946

    # -- construction helper (:114-125) ----------------------------------------------------
    def numerical_clip_alpha(self, log_alphas, clipped_lambda=-5.1):
        """Drop the tail of the table where lambda_t < clipped_lambda (cosine-style schedules)."""
        log_sigmas = 0.5 * torch.log(1. - torch.exp(2. * log_alphas))
        lambs = log_alphas - log_sigmas
        idx = int(torch.searchsorted(torch.flip(lambs, [0]), clipped_lambda))
        if idx > 0:
            log_alphas = log_alphas[:-idx]
        return log_alphas

    def _table(self, device):
        """(t, log_alpha, flipped log_alpha, flipped t) as 1-D tensors on `device` (cached)."""
        key = str(device)
        tab = self._tables.get(key)
        ver = (self.log_alpha_array._version, self.t_array._version)
        if tab is None or tab[4] is not self.log_alpha_array or tab[5] is not self.t_array or tab[6] != ver:
            t = self.t_array.to(device).reshape(-1)
            la = self.log_alpha_array.to(device).reshape(-1)
            tab = (t.contiguous(), la.contiguous(), torch.flip(la, [0]).contiguous(),
                   torch.flip(t, [0]).contiguous(), self.log_alpha_array, self.t_array, ver)
            self._tables[key] = tab
        return tab

    # -- scalar functions (:127-167) ---------------------------------------------------------
    def marginal_log_mean_coeff(self, t):
        """log(alpha_t) for continuous-time labels t (any shape; flattened like the reference)."""
        if self.schedule == "discrete":
            tt, la = self._table(t.device)[:2]
            return _piecewise_linear(t.reshape(-1), tt, la)
        elif self.schedule == "linear":
            return -0.25 * t ** 2 * (self.beta_1 - self.beta_0) - 0.5 * t * self.beta_0
        else:
            import math
            log_alpha_fn = lambda s: torch.log(torch.cos((s + self.cosine_s) / (1. + self.cosine_s) * math.pi / 2.))
            return log_alpha_fn(t) - self.cosine_log_alpha_0

    def marginal_alpha(self, t):
        return torch.exp(self.marginal_log_mean_coeff(t))

    def marginal_std(self, t):
        return torch.sqrt(1. - torch.exp(2. * self.marginal_log_mean_coeff(t)))

    def marginal_lambda(self, t):
        log_mean_coeff = self.marginal_log_mean_coeff(t)
        log_std = 0.5 * torch.log(1. - torch.exp(2. * log_mean_coeff))
        return log_mean_coeff - log_std

    def inverse_lambda(self, lamb):
        """t(lambda): closed form for 'linear' (:161-163), table inversion for 'discrete' (:165-166)."""
        if self.schedule == "linear":
            tmp = 2. * (self.beta_1 - self.beta_0) * torch.logaddexp(-2. * lamb, torch.zeros((1,)).to(lamb))
            Delta = self.beta_0 ** 2 + tmp
            return tmp / (torch.sqrt(Delta) + self.beta_0) / (self.beta_1 - self.beta_0)
        elif self.schedule == "discrete":
            log_alpha = -0.5 * torch.logaddexp(torch.zeros((1,)).to(lamb.device), -2. * lamb)
            la_f, t_f = self._table(lamb.device)[2:4]
            return _piecewise_linear(log_alpha.reshape(-1), la_f, t_f)
        else:
            import math
            log_alpha = -0.5 * torch.logaddexp(-2. * lamb, torch.zeros((1,)).to(lamb))
            t_fn = lambda la: torch.arccos(torch.exp(la + self.cosine_log_alpha_0)) * 2. \
                * (1. + self.cosine_s) / math.pi - self.cosine_s
            return t_fn(log_alpha)


class NoiseScheduleFlow:
    """Flow-matching (rectified-flow) schedule: x_t = alpha_t*x0 + sigma_t*eps on the linear path alpha_t + sigma_t = 1,
    with the time shift of SD3 / FLUX (not in the reference; `schedule == "flow"` is the tag other code switches on):

        sigma_t = shift*t / (1 + (shift - 1)*t),    alpha_t = 1 - sigma_t,    lambda_t = log(alpha_t) - log(sigma_t).

    `model_wrapper(..., model_type="flow")` wraps a network that predicts the velocity v = eps - x0; it receives
    `time_scale * sigma_t` (SD3's convention; time_scale=1 for a network that takes sigma itself). lambda(1) = -inf, so
    sampling starts at T = 1 - 1/total_N and, by default, ends at 1/total_N.

    Every method is fp32 torch arithmetic on `t` with the python floats `shift`, `shift - 1` (formed in double) and
    `time_scale` as scalar operands, in exactly this order (the device controller of the adaptive solver and the tests
    restate it):

        sigma  = (shift * t) / (1. + (shift - 1.) * t)          # shift == 1: (1*t) / (1 + 0*t) == t exactly
        alpha  = 1. - sigma
        log_alpha = log(alpha);   lambda = log_alpha - log(sigma)
        inverse_lambda: sigma = 1. / (1. + exp(lambda));   t = sigma / (shift - (shift - 1.) * sigma)
        model input time = time_scale * sigma
    """

    schedule = "flow"

    def __init__(self, shift=1.0, time_scale=1000.0, total_N=1000):
        shift, time_scale = float(shift), float(time_scale)
        if not shift > 0 or shift == float("inf"):
            raise ValueError("NoiseScheduleFlow: shift must be a positive finite number, got {}".format(shift))
        if int(total_N) != total_N or total_N < 2:
            raise ValueError("NoiseScheduleFlow: total_N must be an integer >= 2, got {}".format(total_N))
        self.shift = shift
        self.time_scale = time_scale
        self.total_N = int(total_N)
        self.T = 1. - 1. / self.total_N

    def marginal_std(self, t):
        return (self.shift * t) / (1. + (self.shift - 1.) * t)

    def marginal_alpha(self, t):
        return 1. - self.marginal_std(t)

    def marginal_log_mean_coeff(self, t):
        return torch.log(self.marginal_alpha(t))

    def marginal_lambda(self, t):
        return self.marginals(t)[2]

    def marginals(self, t):
        """(log_alpha, sigma, lambda, alpha) of a vector of times in one pass (plan.Marginals). The update formulas take
        exp(log_alpha) where the reference's do (:567); alpha itself converts the network output."""
        sigma = self.marginal_std(t)
        alpha = 1. - sigma
        log_alpha = torch.log(alpha)
        return log_alpha, sigma, log_alpha - torch.log(sigma), alpha

    def inverse_lambda(self, lamb):
        sigma = 1. / (1. + torch.exp(lamb))
        return sigma / (self.shift - (self.shift - 1.) * sigma)

    def model_input_time(self, t):
        """What the network receives for the continuous label t: time_scale * sigma_t."""
        return self.time_scale * self.marginal_std(t)


class NoiseScheduleEDM:
    """Schedule of an EDM-preconditioned network (Karras et al. 2022, "Elucidating the Design Space of Diffusion-Based
    Generative Models"; not in the reference; `schedule == "edm"` is the tag other code switches on). The network is
    the raw F of

        D(x; s) = c_skip(s)*x + c_out(s)*F(c_in(s)*x, c_noise(s)),   x = x0 + s*n,
        c_skip = sd^2/(s^2 + sd^2),  c_out = s*sd/sqrt(s^2 + sd^2),  c_in = 1/sqrt(s^2 + sd^2),  c_noise = ln(s)/4

    with sd = sigma_data. The solver integrates in the network's input space y = c_in(s)*x, where

        y_t = alpha_t*x0 + sigma_t*n,   alpha_t = 1/sqrt(s^2 + sd^2),   sigma_t = s/sqrt(s^2 + sd^2),   lambda_t = -ln s,

    so `model_wrapper(..., model_type="edm")` converts F with two words and no division: x0 = (sd^2*alpha_t)*y +
    (sd*sigma_t)*F and eps = sigma_t*y - (sd*alpha_t)*F. The network receives y and c_noise. Start from
    x_T = marginal_std(T) * randn (that is, c_in*sigma_max*n); denoise_to_zero=True returns D(.; sigma_min) in data
    space, which is how Karras's sampler ends.

    The label t in [1/total_N, 1] maps to s by Karras's ramp over u = (t - 1/N)/(1 - 1/N): t = 1 is sigma_max, t = 1/N
    is sigma_min, and skip_type="time_uniform" between the default ends is Karras's grid.

    Every method is fp32 torch arithmetic on `t` with python-float operands formed in double (c = fl32(1/N), 1 - c,
    sigma_min^(1/rho), sigma_max^(1/rho) - sigma_min^(1/rho), 1/rho, rho, sd^2), in exactly this order:

        u      = (t - c) / (1. - c)
        s      = (smin_r + u * span_r) ** rho                      # smin_r = sigma_min^(1/rho), span_r: the difference
        r      = sqrt(s * s + sd^2)
        alpha  = 1. / r;   sigma = s / r;   log_alpha = -log(r);   lambda = -log(s)
        inverse_lambda: s = exp(-lambda);   u = (s ** (1/rho) - smin_r) / span_r;   t = u * (1. - c) + c
        model input time = 0.25 * log(s)
    """

    schedule = "edm"

    def __init__(self, sigma_min=0.002, sigma_max=80., sigma_data=0.5, rho=7., total_N=1000):
        sigma_min, sigma_max, sigma_data, rho = float(sigma_min), float(sigma_max), float(sigma_data), float(rho)
        if not (0. < sigma_min < sigma_max < float("inf")):
            raise ValueError("NoiseScheduleEDM: need 0 < sigma_min < sigma_max < inf, got sigma_min={}, sigma_max={}"
                             .format(sigma_min, sigma_max))
        if not (0. < sigma_data < float("inf")):
            raise ValueError("NoiseScheduleEDM: sigma_data must be a positive finite number, got {}".format(sigma_data))
        if not (0. < rho < float("inf")):
            raise ValueError("NoiseScheduleEDM: rho must be a positive finite number, got {}".format(rho))
        if int(total_N) != total_N or total_N < 2:
            raise ValueError("NoiseScheduleEDM: total_N must be an integer >= 2, got {}".format(total_N))
        self.sigma_min, self.sigma_max, self.sigma_data, self.rho = sigma_min, sigma_max, sigma_data, rho
        self.total_N = int(total_N)
        self.T = 1.
        self._c = float(torch.tensor(1. / self.total_N, dtype=torch.float32))     # fl32(1/N), the default end label
        self._smin_r = sigma_min ** (1. / rho)
        self._span_r = sigma_max ** (1. / rho) - self._smin_r
        self._sd2 = sigma_data * sigma_data

    def sigma(self, t):
        """Karras's noise level s(t) (the VE sigma of x = x0 + s*n)."""
        u = (t - self._c) / (1. - self._c)
        return (self._smin_r + u * self._span_r) ** self.rho

    def _r(self, s):
        return torch.sqrt(s * s + self._sd2)

    def marginal_alpha(self, t):
        return 1. / self._r(self.sigma(t))

    def marginal_std(self, t):
        s = self.sigma(t)
        return s / self._r(s)

    def marginal_log_mean_coeff(self, t):
        return -torch.log(self._r(self.sigma(t)))

    def marginal_lambda(self, t):
        return -torch.log(self.sigma(t))

    def marginals(self, t):
        """(log_alpha, sigma, lambda, alpha) of a vector of times in one pass (plan.Marginals)."""
        s = self.sigma(t)
        r = self._r(s)
        return -torch.log(r), s / r, -torch.log(s), 1. / r

    def inverse_lambda(self, lamb):
        s = torch.exp(-lamb)
        u = (s ** (1. / self.rho) - self._smin_r) / self._span_r
        return u * (1. - self._c) + self._c

    def model_input_time(self, t):
        """What the network receives for the continuous label t: c_noise = ln(s(t))/4."""
        return 0.25 * torch.log(self.sigma(t))

    def conversion_words(self, alpha, sigma, x0):
        """The two words of DPM_PARAM_EDM at the fp32 marginals (alpha_t, sigma_t): (sd^2*alpha_t, sd*sigma_t) for x0,
        (sigma_t, -sd*alpha_t) for eps. Each is formed in double and rounded to fp32 once."""
        f = lambda v: float(torch.tensor(v, dtype=torch.float64).float())
        if x0:
            return f(self._sd2 * alpha), f(self.sigma_data * sigma)
        return f(sigma), f(-self.sigma_data * alpha)
