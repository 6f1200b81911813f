"""Host-side coefficient plan.

Every DPM-Solver update is `x_t = a*x + c0*T0 + c1*T1 + c2*T2` where the T_j are buffered model
values or differences of them (include/dpm_solver_b200.h, `dpm_form`). This module computes the
scalars (a, c_j, w_j) on the HOST, in fp32, in the reference's operation order
(dpm_solver_pytorch.py:563-588, :616-669, :702-789, :815-851, :871-903), vectorised over all
steps of a run, so that the device executes one fused kernel per step and no exp/log/expm1,
no interpolation and no host<->device sync happens inside the sampling loop.

The arithmetic deliberately goes through the same torch CPU scalar ops the reference uses
(`torch.expm1`, `1. / r`, tensor/python-float promotion ...): the resulting fp32 scalars are
bit-identical to the reference evaluated on CPU. All `t` arguments are 1-D fp32 CPU tensors.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Union

import numpy as np
import torch

from ._lib import FORM_DIFF2, FORM_LIN1, FORM_MS3, FORM_SS3T

Number = Union[float, torch.Tensor]


@dataclass
class Coeffs:
    """Scalars of one launch (python floats holding exact fp32 values, signs folded in)."""
    form: int
    a: float
    c0: float
    c1: float = 0.0
    c2: float = 0.0
    w0: float = 0.0
    w1: float = 0.0
    w2: float = 0.0
    w3: float = 0.0
    w4: float = 0.0
    c0_on_old: bool = False
    order: int = 1
    r_tensor: int = 0   # SS3T: bit 0 / 1 = r1 / r2 came as tensors (matters to reference_rounding only)
    dev: Optional[torch.Tensor] = None   # scalars live in this device block instead (on-device adaptive controller)
    g: float = 0.0      # CFG++ (dpm_step_cfgpp): alpha_t of the update's end time, the weight of G - U; 0 when not asked
    cz: float = 0.0     # SDE-DPM-Solver++ (dpm_step_sde): sigma_t*sqrt(-expm1(-2*eta*h)), the weight of the update's noise


def _cpu(t: torch.Tensor) -> torch.Tensor:
    """Time label(s) as a 1-D CPU tensor (syncs if `t` lives on a device)."""
    if not torch.is_tensor(t):
        t = torch.tensor(t)
    return t.detach().reshape(-1).cpu()


def _f(v: Number, i: int = 0) -> float:
    """i-th scalar as a python float; c_float conversion then rounds exactly like torch's
    python-scalar -> fp32 cast."""
    if torch.is_tensor(v):
        return float(v.reshape(-1)[i]) if v.numel() > 1 else float(v)
    return float(v)


class Marginals:
    """log(alpha), alpha, sigma, lambda of a vector of times (one vectorised pass; for a VP schedule the expressions
    are those of marginal_log_mean_coeff / marginal_std / marginal_lambda / marginal_alpha,
    :127-154, sharing the single evaluation of log(alpha))."""

    def __init__(self, ns, t: Optional[torch.Tensor]):
        if t is None:
            return
        self.t = t
        own = getattr(ns, "marginals", None)      # a schedule that is not VP supplies the four itself (NoiseScheduleFlow)
        if own is not None:
            # alpha_e = marginal_alpha(t) converts network outputs (:438); the update formulas take exp(log alpha) (:567)
            self.log_alpha, self.sigma, self.lam, self.alpha_e = own(t)
            self.alpha = torch.exp(self.log_alpha)
            return
        self.log_alpha = ns.marginal_log_mean_coeff(t)
        e2 = 1. - torch.exp(2. * self.log_alpha)
        self.sigma = torch.sqrt(e2)                           # :146
        self.lam = self.log_alpha - 0.5 * torch.log(e2)       # :153-154
        self.alpha = torch.exp(self.log_alpha)                # :140
        self.alpha_e = self.alpha

    def __getitem__(self, i) -> "Marginals":
        m = Marginals(None, None)
        m.t, m.log_alpha, m.sigma, m.lam, m.alpha = self.t[i], self.log_alpha[i], self.sigma[i], self.lam[i], self.alpha[i]
        m.alpha_e = self.alpha_e[i]
        return m


# ---- order 1 ----------------------------------------------------------------------------------

def first_update(ns, algorithm_type: str, s: torch.Tensor, t: torch.Tensor):
    """Vectorised dpm_solver_first_update scalars (:563-588) -> tensors (a, c0)."""
    return _first(algorithm_type, Marginals(ns, s), Marginals(ns, t))


def _sde(eta: float, h, mt: Marginals):
    """SDE-DPM-Solver++ (eta > 0): (h_eta = (1 + eta)*h, the decay exp(-eta*h) that multiplies a, and the noise weight
    cz = sigma_t*sqrt(-expm1(-2*eta*h))). eta == 0 gives (h, None, None): the ODE coefficients, op for op."""
    if not eta:
        return h, None, None
    return (1. + eta) * h, torch.exp(-eta * h), mt.sigma * torch.sqrt(-torch.expm1(-2. * eta * h))


def _first(algorithm_type: str, ms: Marginals, mt: Marginals, eta: float = 0.0):
    h = mt.lam - ms.lam
    if algorithm_type == "dpmsolver++":
        h, decay, _ = _sde(eta, h, mt)
        phi_1 = torch.expm1(-h)
        a = mt.sigma / ms.sigma
        if decay is not None:
            a = a * decay
        c0 = -(mt.alpha * phi_1)
    else:
        phi_1 = torch.expm1(h)
        a = torch.exp(mt.log_alpha - ms.log_alpha)
        c0 = -(mt.sigma * phi_1)
    return a, c0


def first_update_coeffs(ns, algorithm_type, s, t) -> Coeffs:
    a, c0 = first_update(ns, algorithm_type, _cpu(s), _cpu(t))
    return Coeffs(FORM_LIN1, _f(a), _f(c0), order=1)


# ---- multistep --------------------------------------------------------------------------------

def multistep_second(ns, algorithm_type, solver_type, t_prev_1, t_prev_0, t):
    """multistep_dpm_solver_second_update scalars (:815-851) -> tensors (a, c0, c1, inv_r0)."""
    return _ms2(algorithm_type, solver_type, Marginals(ns, t_prev_1), Marginals(ns, t_prev_0), Marginals(ns, t))


def _ms2(algorithm_type, solver_type, m1: Marginals, m0: Marginals, mt: Marginals, eta: float = 0.0):
    h_0 = m0.lam - m1.lam
    h = mt.lam - m0.lam
    r0 = h_0 / h
    inv_r0 = 1. / r0
    if algorithm_type == "dpmsolver++":
        h, decay, _ = _sde(eta, h, mt)
        phi_1 = torch.expm1(-h)
        a = mt.sigma / m0.sigma
        if decay is not None:
            a = a * decay
        b = mt.alpha * phi_1
        c1 = -(0.5 * b) if solver_type == "dpmsolver" else mt.alpha * (phi_1 / h + 1.)
    else:
        phi_1 = torch.expm1(h)
        a = torch.exp(mt.log_alpha - m0.log_alpha)
        b = mt.sigma * phi_1
        c1 = -(0.5 * b) if solver_type == "dpmsolver" else -(mt.sigma * (phi_1 / h - 1.))
    return a, -b, c1, inv_r0


def multistep_third(ns, algorithm_type, t_prev_2, t_prev_1, t_prev_0, t):
    """multistep_dpm_solver_third_update scalars (:871-903); solver_type is ignored there."""
    return _ms3(algorithm_type, *(Marginals(ns, v) for v in (t_prev_2, t_prev_1, t_prev_0, t)))


def _ms3(algorithm_type, m2: Marginals, m1: Marginals, m0: Marginals, mt: Marginals, eta: float = 0.0):
    h_1 = m1.lam - m2.lam
    h_0 = m0.lam - m1.lam
    h = mt.lam - m0.lam
    r0, r1 = h_0 / h, h_1 / h
    w0, w1 = 1. / r0, 1. / r1
    w2 = r0 / (r0 + r1)
    w3 = 1. / (r0 + r1)
    if algorithm_type == "dpmsolver++":
        h, decay, _ = _sde(eta, h, mt)
        phi_1 = torch.expm1(-h)
        phi_2 = phi_1 / h + 1.
        phi_3 = phi_2 / h - 0.5
        a = mt.sigma / m0.sigma
        if decay is not None:
            a = a * decay
        c0, c1, c2 = -(mt.alpha * phi_1), mt.alpha * phi_2, -(mt.alpha * phi_3)
    else:
        phi_1 = torch.expm1(h)
        phi_2 = phi_1 / h - 1.
        phi_3 = phi_2 / h - 0.5
        a = torch.exp(mt.log_alpha - m0.log_alpha)
        c0, c1, c2 = -(mt.sigma * phi_1), -(mt.sigma * phi_2), -(mt.sigma * phi_3)
    return a, c0, c1, c2, w0, w1, w2, w3


def multistep_coeffs(ns, algorithm_type, solver_type, order, t_prev_list, t) -> Coeffs:
    """Scalars of one multistep update of the given order (direct-call path)."""
    tp = [_cpu(v) for v in t_prev_list]
    t = _cpu(t)
    if order == 1:
        return first_update_coeffs(ns, algorithm_type, tp[-1], t)
    if order == 2:
        a, c0, c1, w0 = multistep_second(ns, algorithm_type, solver_type, tp[-2], tp[-1], t)
        return Coeffs(FORM_DIFF2, _f(a), _f(c0), _f(c1), w0=_f(w0), order=2)
    if order == 3:
        v = multistep_third(ns, algorithm_type, tp[-3], tp[-2], tp[-1], t)
        return Coeffs(FORM_MS3, *(_f(u) for u in v[:4]), w0=_f(v[4]), w1=_f(v[5]), w2=_f(v[6]),
                      w3=_f(v[7]), order=3)
    raise ValueError("Solver order must be 1 or 2 or 3, got {}".format(order))


def multistep_orders(steps: int, order: int, lower_order_final: bool) -> List[int]:
    """Order used at update `step` = 1..steps (sample() :1185-1201)."""
    out = []
    for step in range(1, steps + 1):
        if step < order:
            out.append(step)
        elif lower_order_final and steps < 10:
            out.append(min(order, steps + 1 - step))
        else:
            out.append(order)
    return out


def multistep_plan(ns, algorithm_type, solver_type, timesteps: torch.Tensor, order: int,
                   lower_order_final: bool, marginals: Optional[Marginals] = None, cfg_pp: bool = False,
                   eta: float = 0.0) -> List[Coeffs]:
    """Coefficients of every update of a multistep run; plan[i] moves timesteps[i] -> [i+1].
    One vectorised evaluation of the schedule over the grid, then one vector op set per order.
    cfg_pp=True (dpmsolver++, orders 1 and 2): each update also carries g = alpha_t of its end time, the fp32 alpha its
    c0 = -(alpha_t*phi_1) is formed from.
    eta > 0 (dpmsolver++ only): SDE-DPM-Solver++ -- h_eta = (1 + eta)*h in every phi, a multiplied by exp(-eta*h), and
    each update carries cz = sigma_t*sqrt(-expm1(-2*eta*h)), the weight of its Gaussian noise."""
    ts = _cpu(timesteps)
    steps = ts.numel() - 1
    M = marginals if marginals is not None else Marginals(ns, ts)
    orders = multistep_orders(steps, order, lower_order_final)
    plan: List[Optional[Coeffs]] = [None] * steps
    idx = {p: [i for i, o in enumerate(orders) if o == p] for p in (1, 2, 3)}
    if idx[1]:
        i = torch.tensor(idx[1])
        a, c0 = (v.reshape(-1).tolist() for v in _first(algorithm_type, M[i], M[i + 1], eta))
        for k, j in enumerate(idx[1]):
            plan[j] = Coeffs(FORM_LIN1, a[k], c0[k], order=1)
    if idx[2]:
        i = torch.tensor(idx[2])
        a, c0, c1, w0 = (v.reshape(-1).tolist() for v in _ms2(algorithm_type, solver_type, M[i - 1], M[i], M[i + 1], eta))
        for k, j in enumerate(idx[2]):
            plan[j] = Coeffs(FORM_DIFF2, a[k], c0[k], c1[k], w0=w0[k], order=2)
    if cfg_pp:
        g = M.alpha.reshape(-1).tolist()
        for j in idx[1] + idx[2]:
            plan[j].g = g[j + 1]
    if idx[3]:
        i = torch.tensor(idx[3])
        v = [u.reshape(-1).tolist() for u in _ms3(algorithm_type, M[i - 2], M[i - 1], M[i], M[i + 1], eta)]
        for k, j in enumerate(idx[3]):
            plan[j] = Coeffs(FORM_MS3, v[0][k], v[1][k], v[2][k], v[3][k], w0=v[4][k], w1=v[5][k], w2=v[6][k],
                             w3=v[7][k], order=3)
    if eta:
        j = torch.arange(steps)
        cz = _sde(eta, M.lam[j + 1] - M.lam[j], M[j + 1])[2].reshape(-1).tolist()
        for k in range(steps):
            plan[k].cz = cz[k]
    return plan  # type: ignore[return-value]


# ---- singlestep -------------------------------------------------------------------------------

@dataclass
class SinglestepPlan:
    """One outer singlestep update s -> t of order 1, 2 or 3."""
    order: int
    times: List[torch.Tensor]        # model evaluation times: [s] / [s, s1] / [s, s1, s2] (CPU, (1,))
    stages: List[Coeffs] = field(default_factory=list)  # one launch per model evaluation


def singlestep_second(ns, algorithm_type, solver_type, s, t, r1: Number = 0.5) -> SinglestepPlan:
    """singlestep_dpm_solver_second_update scalars (:613-669)."""
    if r1 is None:
        r1 = 0.5
    s, t = _cpu(s), _cpu(t)
    ms, mt = Marginals(ns, s), Marginals(ns, t)
    h = mt.lam - ms.lam
    s1 = ns.inverse_lambda(ms.lam + r1 * h)
    m1 = Marginals(ns, s1)
    if algorithm_type == "dpmsolver++":
        phi_11 = torch.expm1(-r1 * h)
        phi_1 = torch.expm1(-h)
        st1 = Coeffs(FORM_LIN1, _f(m1.sigma / ms.sigma), _f(-(m1.alpha * phi_11)), order=2)
        b = mt.alpha * phi_1
        if solver_type == "dpmsolver":
            c1 = -((0.5 / r1) * b)
        else:
            c1 = (1. / r1) * (mt.alpha * (phi_1 / h + 1.))
        fin = Coeffs(FORM_DIFF2, _f(mt.sigma / ms.sigma), _f(-b), _f(c1), w0=1.0, c0_on_old=True, order=2)
    else:
        phi_11 = torch.expm1(r1 * h)
        phi_1 = torch.expm1(h)
        st1 = Coeffs(FORM_LIN1, _f(torch.exp(m1.log_alpha - ms.log_alpha)), _f(-(m1.sigma * phi_11)), order=2)
        b = mt.sigma * phi_1
        if solver_type == "dpmsolver":
            c1 = -((0.5 / r1) * b)
        else:
            c1 = -((1. / r1) * (mt.sigma * (phi_1 / h - 1.)))
        fin = Coeffs(FORM_DIFF2, _f(torch.exp(mt.log_alpha - ms.log_alpha)), _f(-b), _f(c1), w0=1.0,
                     c0_on_old=True, order=2)
    return SinglestepPlan(2, [s, s1], [st1, fin])


def singlestep_third(ns, algorithm_type, solver_type, s, t, r1: Number = 1. / 3.,
                     r2: Number = 2. / 3.) -> SinglestepPlan:
    """singlestep_dpm_solver_third_update scalars (:697-789)."""
    if r1 is None:
        r1 = 1. / 3.
    if r2 is None:
        r2 = 2. / 3.
    rt = (1 if torch.is_tensor(r1) else 0) | (2 if torch.is_tensor(r2) else 0)
    s, t = _cpu(s), _cpu(t)
    ms, mt = Marginals(ns, s), Marginals(ns, t)
    h = mt.lam - ms.lam
    s1 = ns.inverse_lambda(ms.lam + r1 * h)
    s2 = ns.inverse_lambda(ms.lam + r2 * h)
    m1, m2 = Marginals(ns, s1), Marginals(ns, s2)
    pp = algorithm_type == "dpmsolver++"
    if pp:
        phi_11 = torch.expm1(-r1 * h)
        phi_12 = torch.expm1(-r2 * h)
        phi_1 = torch.expm1(-h)
        phi_22 = torch.expm1(-r2 * h) / (r2 * h) + 1.
        phi_2 = phi_1 / h + 1.
        phi_3 = phi_2 / h - 0.5
        a1, a2, at = m1.sigma / ms.sigma, m2.sigma / ms.sigma, mt.sigma / ms.sigma
        g1, g2, gt = m1.alpha, m2.alpha, mt.alpha
        st1 = Coeffs(FORM_LIN1, _f(a1), _f(-(g1 * phi_11)), order=3)
        st2 = Coeffs(FORM_DIFF2, _f(a2), _f(-(g2 * phi_12)), _f(r2 / r1 * (g2 * phi_22)), w0=1.0,
                     c0_on_old=True, order=3)
        if solver_type == "dpmsolver":
            fin = Coeffs(FORM_DIFF2, _f(at), _f(-(gt * phi_1)), _f((1. / r2) * (gt * phi_2)), w0=1.0,
                         c0_on_old=True, order=3)
        else:
            fin = Coeffs(FORM_SS3T, _f(at), _f(-(gt * phi_1)), _f(gt * phi_2), _f(-(gt * phi_3)),
                         w0=_f(1. / r1), w1=_f(1. / r2), w2=_f(r2), w3=_f(r1), w4=_f(r2 - r1), order=3, r_tensor=rt)
    else:
        phi_11 = torch.expm1(r1 * h)
        phi_12 = torch.expm1(r2 * h)
        phi_1 = torch.expm1(h)
        phi_22 = torch.expm1(r2 * h) / (r2 * h) - 1.
        phi_2 = phi_1 / h - 1.
        phi_3 = phi_2 / h - 0.5
        a1 = torch.exp(m1.log_alpha - ms.log_alpha)
        a2 = torch.exp(m2.log_alpha - ms.log_alpha)
        at = torch.exp(mt.log_alpha - ms.log_alpha)
        g1, g2, gt = m1.sigma, m2.sigma, mt.sigma
        st1 = Coeffs(FORM_LIN1, _f(a1), _f(-(g1 * phi_11)), order=3)
        st2 = Coeffs(FORM_DIFF2, _f(a2), _f(-(g2 * phi_12)), _f(-(r2 / r1 * (g2 * phi_22))), w0=1.0,
                     c0_on_old=True, order=3)
        if solver_type == "dpmsolver":
            fin = Coeffs(FORM_DIFF2, _f(at), _f(-(gt * phi_1)), _f(-((1. / r2) * (gt * phi_2))), w0=1.0,
                         c0_on_old=True, order=3)
        else:
            fin = Coeffs(FORM_SS3T, _f(at), _f(-(gt * phi_1)), _f(-(gt * phi_2)), _f(-(gt * phi_3)),
                         w0=_f(1. / r1), w1=_f(1. / r2), w2=_f(r2), w3=_f(r1), w4=_f(r2 - r1), order=3, r_tensor=rt)
    return SinglestepPlan(3, [s, s1, s2], [st1, st2, fin])


def singlestep_plan(ns, algorithm_type, solver_type, order, s, t, r1=None, r2=None) -> SinglestepPlan:
    if order == 1:
        s = _cpu(s)
        return SinglestepPlan(1, [s], [first_update_coeffs(ns, algorithm_type, s, t)])
    if order == 2:
        return singlestep_second(ns, algorithm_type, solver_type, s, t, r1)
    if order == 3:
        return singlestep_third(ns, algorithm_type, solver_type, s, t, r1, r2)
    raise ValueError("Solver order must be 1 or 2 or 3, got {}".format(order))


def singlestep_orders(steps: int, order: int) -> List[int]:
    """Orders of 'DPM-Solver-fast' for a budget of `steps` evaluations (:514-533)."""
    if order == 3:
        K = steps // 3 + 1
        if steps % 3 == 0:
            return [3, ] * (K - 2) + [2, 1]
        elif steps % 3 == 1:
            return [3, ] * (K - 1) + [1]
        return [3, ] * (K - 1) + [2]
    if order == 2:
        if steps % 2 == 0:
            return [2, ] * (steps // 2)
        return [2, ] * (steps // 2) + [1]
    if order == 1:
        return [1, ] * steps
    raise ValueError("'order' must be '1' or '2' or '3'.")


# ---- UniPC multistep (unipc.py) ----------------------------------------------------------------

@dataclass
class UniCoeffs:
    """Words of one dpm_step_unipc launch (python floats holding exact fp32 values, signs folded in): the corrector of
    step i (order pc, 0 = off) and the predictor of step i+1 (order pp, 0 = none)."""
    pc: int
    pp: int
    cd: tuple = (0.0, 0.0)
    ct: float = 0.0
    a: float = 0.0
    c0: float = 0.0
    cp: tuple = (0.0, 0.0)
    form: int = FORM_LIN1       # (the descriptor's form: not read by dpm_step_unipc)
    order: int = 0

    def corrector_only(self) -> "UniCoeffs":
        return UniCoeffs(self.pc, 0, self.cd, self.ct, order=self.order)

    def predictor_only(self) -> "UniCoeffs":
        return UniCoeffs(0, self.pp, a=self.a, c0=self.c0, cp=self.cp, order=self.order)


def unipc_orders(steps: int, order: int, lower_order_final: bool) -> List[int]:
    """Order p_i of UniPC step i = 1..steps: min(order, i), capped at steps + 1 - i with lower_order_final (for every
    `steps`, unlike DPM_Solver's multistep rule, which lowers the final orders only when steps < 10)."""
    return [min(order, i, steps + 1 - i) if lower_order_final else min(order, i) for i in range(1, steps + 1)]


def _g(x: float, j: int) -> float:
    """(e^x - sum_{m<=j} x^m/m!) / x^j in fp64: the series for |x| < 0.5, where the direct form cancels."""
    if abs(x) < 0.5:
        s, term = 0.0, 1.0
        for m in range(j + 1, j + 30):
            term = x ** (m - j) / math.factorial(m)
            s += term
        return s
    return (math.expm1(x) - sum(x ** m / math.factorial(m) for m in range(1, j + 1))) / x ** j


def unipc_step_weights(lam: List[float], i: int, p: int, pp_alg: bool, bh2: bool):
    """fp64 scalars of UniPC step i (lam: the grid's lambda values): (hh, B, r[1..p], rho_p, rho_c)."""
    h = lam[i] - lam[i - 1]
    hh = -h if pp_alg else h
    B = math.expm1(hh) if bh2 else hh
    r = [(lam[i - 1 - k] - lam[i - 1]) / h for k in range(1, p)] + [1.0]
    # b_j = h_phi_k * j! / B with h_phi_k = g_j(hh) after j - 1 steps of the recursion h_phi_k/hh - 1/f
    b = [_g(hh, j) * math.factorial(j) / B for j in range(1, p + 1)]
    R = [[rk ** (j - 1) for rk in r] for j in range(1, p + 1)]
    if p == 1:
        rho_p = []
    elif p == 2:
        rho_p = [0.5]
    else:
        rho_p = list(np.linalg.solve(np.array(R)[:p - 1, :p - 1], np.array(b[:p - 1])))
    rho_c = [0.5] if p == 1 else list(np.linalg.solve(np.array(R), np.array(b)))
    return hh, B, r, rho_p, rho_c


def unipc_plan(algorithm_type: str, variant: str, marg: Marginals, orders: List[int], use_corrector: bool):
    """(LIN1 Coeffs of step 1's predictor, [UniCoeffs of launches 1..N-1]). Every word is evaluated in fp64 from the
    fp32 marginals and rounded to fp32 once."""
    pp_alg, bh2 = algorithm_type == "dpmsolver++", variant == "bh2"
    lam = marg.lam.double().tolist()
    al = marg.alpha.double().tolist()
    sg = marg.sigma.double().tolist()
    N = len(orders)
    f = lambda v: float(np.float32(v))
    a1, c01 = _first(algorithm_type, marg[torch.tensor([0])], marg[torch.tensor([1])])
    first = Coeffs(FORM_LIN1, _f(a1), _f(c01), order=1)
    scale = sg if not pp_alg else al             # alpha_i for data prediction, sigma_i for noise prediction
    W = [None] + [unipc_step_weights(lam, i, orders[i - 1], pp_alg, bh2) for i in range(1, N + 1)]
    launches = []
    for i in range(1, N):
        p, q = orders[i - 1], orders[i]
        _, B, r, rho_p, rho_c = W[i]
        cd, ct, pc = [0.0, 0.0], 0.0, 0
        if use_corrector:
            pc = p
            for k in range(1, p):
                cd[k - 1] = f(-scale[i] * B * (rho_c[k - 1] - rho_p[k - 1]) / r[k - 1])
            ct = f(-scale[i] * B * rho_c[p - 1])
        hh2, B2, r2, rho_p2, _ = W[i + 1]
        a = sg[i + 1] / sg[i] if pp_alg else al[i + 1] / al[i]
        cp = [0.0, 0.0]
        for k in range(1, q):
            cp[k - 1] = f(-scale[i + 1] * B2 * rho_p2[k - 1] / r2[k - 1])
        launches.append(UniCoeffs(pc, q, tuple(cd), ct, f(a), f(-scale[i + 1] * math.expm1(hh2)), tuple(cp), order=q))
    return first, launches
