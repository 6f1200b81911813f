"""Oracles of adaptive projected guidance (model_wrapper's apg_eta) -- TEST INFRASTRUCTURE.

* `apg_fp64`: the method in float64, written from the paper's formulas (Sadat, Hilliges and Weber, "Eliminating
  Oversaturation and Artifacts of High Guidance Scales in Diffusion Models", ICLR 2025, Algorithm 1): the guidance
  difference with reverse momentum, norm-clipped, split into the part parallel to the normalised conditional prediction
  and the part orthogonal to it, the parallel part scaled by eta.
* `x0_fp64`: each parameterisation's denoised prediction in float64.
* `APGOracle`: the numpy executor (edm_oracle.EDMOracle: every parameterisation, guidance form and dpm_step_unipc) plus
  dpm_apg_words and dpm_step_apg as include/dpm_solver_b200.h states them, op for op in IEEE fp32, the sums in fp64
  (numpy's pairwise order; `exact=True`: words.cu's order, `apg_words_exact`, so that the words are bit-exact).
* `apg_words_exact`: the words of words.cu operation for operation -- its chunks, thread ownership, warp butterflies,
  warp order, chunk merge and k_apg_final's left-to-right fp64 formula.
* `reference_solver`: the UNMODIFIED reference DPM_Solver driven by an fp64 APG data-prediction function, with the
  momentum kept in its closure.
"""
import numpy as np
import torch

from edm_oracle import EDMOracle
from oracle import ref_loader
from oracle_backend import _np

f32 = np.float32
PARAM_NOISE, PARAM_X_START, PARAM_V, PARAM_SCORE, PARAM_FLOW, PARAM_EDM = range(6)


# ---- the method in fp64 ----------------------------------------------------------------------------------------------

class APG64:
    """Algorithm 1 of the paper on [B, ...] float64 arrays; `running` is the momentum state across calls."""

    def __init__(self, eta, norm_threshold=0.0, momentum=0.0):
        self.eta, self.r, self.beta = eta, norm_threshold, momentum
        self.running = None

    def __call__(self, c, u, w):
        c, u = np.asarray(c, np.float64), np.asarray(u, np.float64)
        B = c.shape[0]
        diff = c - u
        if self.beta != 0:
            self.running = diff if self.running is None else diff + self.beta * self.running
            diff = self.running
        flat = diff.reshape(B, -1)
        if self.r > 0:
            norm = np.sqrt((flat * flat).sum(axis=1, keepdims=True))
            flat = flat * np.minimum(1.0, self.r / norm)
        v1 = c.reshape(B, -1)
        v1 = v1 / np.maximum(np.sqrt((v1 * v1).sum(axis=1, keepdims=True)), 1e-12)    # F.normalize
        par = (flat * v1).sum(axis=1, keepdims=True) * v1
        orth = flat - par
        update = (orth + self.eta * par).reshape(c.shape)
        w = np.asarray(w, np.float64).reshape((-1,) + (1,) * (c.ndim - 1))
        return c + (w - 1.0) * update


def x0_fp64(param, out, x, alpha, sigma, sigma_data=None):
    """The denoised prediction of one network output in float64 (alpha, sigma: the marginals)."""
    out, x = np.asarray(out, np.float64), np.asarray(x, np.float64)
    if param == PARAM_NOISE:
        return (x - sigma * out) / alpha
    if param == PARAM_X_START:
        return out
    if param == PARAM_V:
        return alpha * x - sigma * out
    if param == PARAM_SCORE:
        return (x + sigma * sigma * out) / alpha
    if param == PARAM_FLOW:
        return x - sigma * out
    if param == PARAM_EDM:
        return sigma_data * sigma_data * alpha * x + sigma_data * sigma * out
    raise ValueError(param)


# ---- words.cu's reduction, operation for operation -------------------------------------------------------------------

CHUNK, THREADS, WARP = 8192, 256, 32


def chunk_sums(v):
    """The CTA sums [B, chunks] of fp64 terms v [B, per_sample] as the words passes form them: CTA (b, chunk) covers
    chunk elements [chunk*8192, min(+8192, per_sample)); thread tid owns the elements (u*256 + tid)*8 + i, u = 0..3,
    i = 0..7, and adds their terms in that order to a sum that starts at 0.0. Each warp folds its 32 lanes by
    v += shfl_xor(v, o), o = 16 .. 1; then s = 0.0 + warp 0 + ... + warp 7. Elements past the end of the sample are
    skipped; here they add +0.0, which leaves every such sum (never -0.0: it starts at +0.0) unchanged."""
    Bn, ps = v.shape
    chunks = -(-ps // CHUNK)
    pad = chunks * CHUNK - ps
    with np.errstate(all="ignore"):
        v = np.concatenate([v, np.zeros((Bn, pad))], axis=1) if pad else v
        # [B, chunk, u, tid, i] -> [B, chunk, tid, (u, i)]: each thread's 32 terms in the order it adds them
        per_thread = v.reshape(Bn, chunks, 4, THREADS, 8).transpose(0, 1, 3, 2, 4).reshape(Bn, chunks, THREADS, 32)
        t = np.zeros((Bn, chunks, THREADS))
        for k in range(32):
            t = t + per_thread[..., k]
        lanes = t.reshape(Bn, chunks, THREADS // WARP, WARP)
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[..., np.arange(WARP) ^ o]
        s = np.zeros((Bn, chunks))
        for w in range(THREADS // WARP):
            s = s + lanes[:, :, w, 0]
    return s


def device_sum(v):
    """The per-sample fp64 sum [B] of the terms v [B, per_sample] in the words passes' order: chunk_sums, merged from
    0.0 in chunk order."""
    s = chunk_sums(v)
    t = np.zeros(s.shape[0])
    with np.errstate(all="ignore"):
        for ch in range(s.shape[1]):
            t = t + s[:, ch]
    return t


def apg_sums_exact(R, c):
    """(||R||^2, <R, c>, ||c||^2) per sample as the APG words pass (ApgPass) + k_apg_final sum them, from fp32
    [B, per_sample] arrays: the device_sum of the fp64 products (the product of two fp32 values is exact in fp64)."""
    R, c = np.asarray(R, f32).astype(np.float64), np.asarray(c, f32).astype(np.float64)
    with np.errstate(all="ignore"):
        return device_sum(R * R), device_sum(R * c), device_sum(c * c)


def apg_final(srr, src, scc, w, eta, norm_threshold):
    """k_apg_final from the merged sums: fp64, left to right, each word rounded to fp32 once -> fp32 [2, B]. `w`: the
    scale of each sample as fp64 (an fp32 value widened)."""
    with np.errstate(all="ignore"):
        k = np.ones(len(srr))
        if f32(norm_threshold) > 0:
            q = np.float64(f32(norm_threshold)) / np.sqrt(srr)
            k = np.where(q < 1.0, q, 1.0)            # (a NaN quotient gives 1, as `q < 1.0 ? q : 1.0` does)
        sc = np.sqrt(scc)
        nc = np.where(sc < 1e-12, 1e-12, sc)
        p = src / (nc * nc)
        A = 1.0 - (((w - 1.0) * (1.0 - np.float64(f32(eta)))) * k) * p
        Bw = (w - 1.0) * k
        return np.stack([A, Bw]).astype(f32)


def apg_words_exact(R, c, w, eta, norm_threshold):
    """The words [2, B] of dpm_apg_words from R and c (fp32 [B, per_sample]) and the per-sample scales `w` (fp64 [B])."""
    return apg_final(*apg_sums_exact(R, c), w, eta, norm_threshold)


# ---- the executor ----------------------------------------------------------------------------------------------------

class APGOracle(EDMOracle):
    """The numpy executor with dpm_apg_words and dpm_step_apg. `exact`: the words summed in words.cu's order
    (apg_words_exact), bit-exact with the device; otherwise in numpy's pairwise order (within an ulp of it)."""

    def __init__(self, exact=False):
        super().__init__()
        self.exact = exact

    @staticmethod
    def _x0(a, out, xe):
        """apg_x0: the step's conversion to x0, each op rounded."""
        al, sg = f32(a.alpha_e), f32(a.sigma_e)
        with np.errstate(all="ignore"):
            if a.param == PARAM_FLOW:
                return (xe - sg * out).astype(f32)
            if a.param == PARAM_EDM:
                return (al * xe + sg * out).astype(f32)
            if a.param == PARAM_X_START:
                eps = (xe - al * out) / sg
            elif a.param == PARAM_V:
                eps = al * out + sg * xe
            elif a.param == PARAM_SCORE:
                eps = (-sg) * out
            else:
                eps = out
            return ((xe - sg * eps) / al).astype(f32)

    def _halves(self, a):
        xe = _np(a.xe if a.xe is not None else a.x)
        c = self._x0(a, _np(a.e_cond), xe)
        return xe, c

    def apg_words(self, a, eta, norm_threshold, momentum, r_prev=None, r_out=None):
        self.launches += 2
        self.log.append(("apg_words", a.n_model))
        xe, c = self._halves(a)
        B = c.shape[0]
        with np.errstate(all="ignore"):
            D = (c - self._x0(a, _np(a.e_uncond), xe)).astype(f32)
            R = D if r_prev is None else (D + f32(momentum) * _np(r_prev)).astype(f32)
        if r_out is not None:
            r_out.copy_(torch.from_numpy(np.ascontiguousarray(R)).reshape(r_out.shape))
        w = (_np(a.guidance_b).astype(np.float64) if a.guidance_b is not None
             else np.full(B, np.float64(f32(a.guidance))))
        if self.exact:
            # the device sums in storage order: a channels_last launch (laid out like xe) holds each sample as (h, w, c)
            ref = a.xe if a.xe is not None else a.x
            if ref.dim() in (4, 5) and not ref.is_contiguous() and ref.is_contiguous(
                    memory_format=torch.channels_last if ref.dim() == 4 else torch.channels_last_3d):
                perm = (0,) + tuple(range(2, ref.dim())) + (1,)
                R, c = R.transpose(perm), c.transpose(perm)
            sums = apg_sums_exact(R.reshape(B, -1), c.reshape(B, -1))
        else:
            R64, c64 = R.reshape(B, -1).astype(np.float64), c.reshape(B, -1).astype(np.float64)
            with np.errstate(all="ignore"):
                sums = (R64 * R64).sum(1), (R64 * c64).sum(1), (c64 * c64).sum(1)
        return torch.from_numpy(apg_final(*sums, w, eta, norm_threshold))

    def _model_value(self, a, thr=None):
        if getattr(a, "apg_words", None) is None:
            return super()._model_value(a, thr)
        xe, c = self._halves(a)
        B = c.shape[0]
        W = _np(a.apg_words).reshape(2, B)
        shape = (B,) + (1,) * (c.ndim - 1)
        A, Bw = W[0].reshape(shape), W[1].reshape(shape)
        with np.errstate(all="ignore"):
            R = _np(a.apg_r) if a.apg_r is not None else (c - self._x0(a, _np(a.e_uncond), xe)).astype(f32)
            g = (A * c + Bw * R).astype(f32)
            if a.guidance_b is not None:
                g = np.where((_np(a.guidance_b) == 1).reshape(shape), c, g)
            if a.predict_x0:
                if thr is not None:
                    s = np.repeat(thr.reshape(-1), a.per_sample).reshape(g.shape)
                    g = np.minimum(np.maximum(g, -s), s) / s
                return g.astype(f32)
            return ((xe - f32(a.alpha_t) * g) / f32(a.sigma_t)).astype(f32)


# ---- the reference driven by an fp64 APG data prediction ---------------------------------------------------------------

def apg_x0_model(net, ns, param, uc, c, w, eta, norm_threshold=0.0, momentum=0.0, input_time=None):
    """x0_fn(x, t) -> the APG-guided denoised prediction in float64 (returned as fp32): the network runs on
    cat([x, x]) with cat([uc, c]) as model_wrapper runs it; `ns` gives the fp32 marginals at t; momentum is kept in the
    closure across calls (one closure per sample() run)."""
    apg = APG64(eta, norm_threshold, momentum)
    sd = getattr(ns, "sigma_data", None)

    def fn(x, t):
        t_in = input_time(t) if input_time is not None else t
        out_u, out_c = net(torch.cat([x, x]), torch.cat([t_in, t_in]), torch.cat([uc, c])).chunk(2)
        al = ns.marginal_alpha(t).double().numpy().reshape((-1,) + (1,) * (x.dim() - 1))
        sg = ns.marginal_std(t).double().numpy().reshape(al.shape)
        xn = x.double().numpy()
        cx = x0_fp64(param, out_c.double().numpy(), xn, al, sg, sd)
        ux = x0_fp64(param, out_u.double().numpy(), xn, al, sg, sd)
        return torch.from_numpy(apg(cx, ux, w)).float()
    return fn


def reference_solver(ns, x0_fn, algorithm_type, thresholding=False):
    """The unmodified reference DPM_Solver whose data prediction is x0_fn and whose noise prediction is the x_start
    conversion of it, (x - alpha_t*x0)/sigma_t in eager torch (:292)."""
    ref = ref_loader.load("dpm_solver_pytorch")

    class APGSolver(ref.DPM_Solver):
        def data_prediction_fn(self, x, t):
            x0 = x0_fn(x, t.expand((x.shape[0])))
            return x0 if self.correcting_x0_fn is None else self.correcting_x0_fn(x0, t)

        def noise_prediction_fn(self, x, t):
            x0 = x0_fn(x, t.expand((x.shape[0])))
            return (x - self.noise_schedule.marginal_alpha(t) * x0) / self.noise_schedule.marginal_std(t)

    return APGSolver(lambda x, t: None, ns, algorithm_type=algorithm_type,
                     correcting_x0_fn="dynamic_thresholding" if thresholding else None)
