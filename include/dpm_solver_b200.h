/*
 * dpm_solver_b200.h -- C-ABI of libdpmsolver_b200.so
 *
 * H100 (sm_90a) implementation of DPM-Solver's per-step update path. The reference
 * (LuChengTHU/dpm-solver, dpm_solver_pytorch.py) has no FFI: every function below replaces a
 * run of PyTorch eager elementwise ops in that file; the line ranges are cited per function.
 *
 * Conventions
 *   - all tensor arguments are raw DEVICE pointers to contiguous memory, `n` elements;
 *   - scalars (alpha, sigma, phi, ... ) are fp32 computed on the HOST and passed by value, so
 *     every launch is CUDA-graph capturable and no exp/log runs per element on the device;
 *   - arithmetic is fp32 in registers in the reference's exact operation order with FMA
 *     contraction disabled (results are bit-identical to the reference's fp32 CPU path when the
 *     storage dtype is fp32); bf16/f16 storage is rounded to nearest-even once, on store;
 *   - inputs are read-only and may alias each other; `out` may alias `x` (element-wise
 *     in-place) but no other overlap is allowed;
 *   - every entry point takes the stream explicitly, never synchronises, never allocates;
 *   - return value: 0 on success, negative dpm_status on argument errors, positive cudaError_t
 *     on CUDA errors. dpm_last_error() returns a thread-local description.
 */
#ifndef DPM_SOLVER_B200_H
#define DPM_SOLVER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DPM_B200_VERSION 108 /* 0.1.8: CFG++ (dpm_step_cfgpp); regional guidance (dpm_step_multi_masked), TCFG
                                (dpm_tcfg_words, dpm_step_tcfg) and frequency-decoupled guidance (dpm_fdg_supported,
                                dpm_fdg_guided), Perp-Neg (dpm_perpneg_workspace, dpm_perpneg_words) and
                                SDE-DPM-Solver++ (dpm_step_sde) are additions to this ABI: test for their symbols */

#if defined(__GNUC__)
#define DPM_API __attribute__((visibility("default")))
#else
#define DPM_API
#endif

typedef void* dpm_stream_t; /* cudaStream_t */

typedef enum dpm_status {
  DPM_OK = 0,
  DPM_ERR_ARG = -1,         /* null pointer / bad enum / bad size */
  DPM_ERR_UNSUPPORTED = -2, /* valid request this build cannot serve */
  DPM_ERR_ALIGN = -3        /* reserved: (mis)alignment is handled internally today */
} dpm_status;

typedef enum dpm_dtype { DPM_F32 = 0, DPM_BF16 = 1, DPM_F16 = 2 } dpm_dtype;

/* How the buffered "model value" T0 and the older buffers enter the update.
 * NEW = the most recent model value (computed in-kernel from raw model outputs when
 * n_model > 0, else loaded from m0); M1/M2 = older buffers.
 *
 *   NONE : no state update, only m_out is written (data_prediction_fn :433-442)
 *   LIN1 : out = a*x + c0*NEW                                   (first update :573-588)
 *   LIN2 : out = a*x + c0*NEW + c1*M1                           (generic AXPY chains)
 *   LIN3 : out = a*x + c0*NEW + c1*M1 + c2*M2
 *   DIFF2: D = w0*(NEW - M1); out = a*x + c0*(c0_on_old ? M1 : NEW) + c1*D
 *          multistep-2 :823-851 (c0_on_old=0, w0=1/r0) and the singlestep difference
 *          steps :630-669, :728-739, :767-778 (c0_on_old=1, w0=1, M1 = model_s)
 *   MS3  : D10=w0*(NEW-M1); D11=w1*(M1-M2); dd=D10-D11; D1=D10+w2*dd; D2=w3*dd;
 *          out = a*x + c0*NEW + c1*D1 + c2*D2                   (multistep-3 :880-903)
 *   SS3T : singlestep-3 'taylor' :741-750 / :780-789, M2=model_s, M1=model_s1, NEW=model_s2:
 *          D10=w0*(M1-M2); D11=w1*(NEW-M2); D1=(w2*D10-w3*D11)/w4; D2=(2*(D11-D10))/w4;
 *          out = a*x + c0*M2 + c1*D1 + c2*D2
 * Sums are evaluated left to right, each product and each sum rounded separately.
 */
typedef enum dpm_form {
  DPM_FORM_NONE = 0,
  DPM_FORM_LIN1 = 1,
  DPM_FORM_LIN2 = 2,
  DPM_FORM_LIN3 = 3,
  DPM_FORM_DIFF2 = 4,
  DPM_FORM_MS3 = 5,
  DPM_FORM_SS3T = 6
} dpm_form;

/* Parameterisation of the network output, model_wrapper.noise_pred_fn :288-298.
 * DPM_PARAM_FLOW (not in the reference): the velocity v = eps - x0 of a flow-matching model on the linear path
 * x_t = alpha_t*x0 + sigma_t*eps with alpha_t + sigma_t = 1. Its conversion lands directly in the solver's space, two
 * separately rounded ops and no division:
 *   predict_x0 == 1 : x0  = xe - sigma_e*out      (the eps -> x0 division :439 is skipped; the clamp follows)
 *   predict_x0 == 0 : eps = xe + alpha_e*out
 * DPM_PARAM_EDM (not in the reference): the raw network F of an EDM-preconditioned model (Karras et al. 2022),
 * D(x; s) = c_skip*x + c_out*F(c_in*x, c_noise), integrated in the network's input space y = c_in*x. alpha_e and
 * sigma_e then carry two host-computed words instead of the marginals, and the conversion is one affine map in either
 * space, three separately rounded ops and no division:
 *   value = alpha_e*xe + sigma_e*out
 *   predict_x0 == 1 : words (sd^2*alpha_t, sd*sigma_t)  -> x0   (the eps -> x0 division :439 is skipped)
 *   predict_x0 == 0 : words (sigma_t, -sd*alpha_t)       -> eps
 * Classifier-free guidance in every form converts each output so and combines the converted values
 * (T = T_u + s*(T_c - T_u)); a rescaled step combines and rescales the raw outputs, then converts. */
typedef enum dpm_param {
  DPM_PARAM_NOISE = 0,   /* eps = out                         :289 */
  DPM_PARAM_X_START = 1, /* eps = (xe - alpha*out)/sigma      :292 */
  DPM_PARAM_V = 2,       /* eps = alpha*out + sigma*xe        :295 */
  DPM_PARAM_SCORE = 3,   /* eps = (-sigma)*out                :298 */
  DPM_PARAM_FLOW = 4,    /* x0 = xe - sigma*out  or  eps = xe + alpha*out (see above) */
  DPM_PARAM_EDM = 5      /* alpha*xe + sigma*out, alpha / sigma the words above      */
} dpm_param;

/* One fused solver step. With n_model == 0 this is a pure update on buffered model values.
 * With n_model >= 1 it is the fused "post-model" step: raw network outputs are converted to
 * the buffered model value (parameterisation -> CFG combine -> eps->x0 -> thresholding
 * clamp), optionally stored to m_out, and consumed by the update in the same pass. */
typedef struct dpm_step_desc {
  /* state dtype tensors */
  const void* x;   /* base state x_s of the update (may be NULL iff form == NONE)          */
  const void* xe;  /* state the model was evaluated at (== x for multistep; x_s1/x_s2 for
                      singlestep); used by x_start/v conversion and eps->x0. NULL => x    */
  const void* m0;  /* NEW buffered model value, read when n_model == 0                      */
  const void* m1;  /* older buffers, as the form requires                                  */
  const void* m2;
  void* m_out;     /* optional: computed model value written here (n_model >= 1)           */
  void* out;       /* x_t; required unless form == NONE                                    */
  void* out2;      /* optional second copy of x_t (e.g. the other half of the network's
                      doubled CFG batch, model_wrapper :326); NULL = none                   */
  /* model dtype tensors */
  const void* e_cond;   /* network output (conditional half under CFG)                     */
  const void* e_uncond; /* unconditional half, n_model == 2; CFG :329-330                  */
  /* per-sample thresholds s_b (already max'ed with thresholding_max_val), fp32 [n/per_sample]
   * or NULL. clamp(x0,-s,s)/s, dynamic_thresholding_fn :423-424 */
  const float* thr;
  uint64_t n;          /* total elements                                                   */
  uint64_t per_sample; /* elements per sample (C*H*W); read when thr != NULL, and by the masked step */
  int32_t state_dtype; /* dpm_dtype of x, xe, m*, m_out, out                               */
  int32_t model_dtype; /* dpm_dtype of e_cond, e_uncond                                    */
  int32_t form;        /* dpm_form                                                         */
  int32_t n_model;     /* 0, 1 or 2 raw network outputs                                    */
  int32_t param;       /* dpm_param                                                        */
  int32_t predict_x0;  /* 1: buffered value is x0 = (xe - sigma_e*eps)/alpha_e :439 (FLOW, EDM: see there) */
  int32_t c0_on_old;   /* DIFF2 only                                                       */
  int32_t raw_round;   /* 0 (default). Reference-rounding mode for networks that return 16-bit NOISE into an
                          fp32 state: bits 0-1 = DPM_BF16 / DPM_F16, the type the raw outputs arrived in --
                          the CFG combine :329-330 then rounds to it after each of its three ops, as the
                          reference's eager 16-bit ops do; bit 2 (+4) = the buffered values are such raw
                          outputs, so their differences (:823, :880-881, :636, :735, :741-742) are rounded
                          to that type before the fp32 coefficients widen them. Served by the vector
                          kernels for bf16 / f16 network outputs, else by the generic kernel.          */
  float guidance;      /* CFG scale s: eps = eps_u + s*(eps_c - eps_u) :330                */
  float alpha_e;       /* alpha, sigma at the model evaluation time (DPM_PARAM_EDM: its two words) */
  float sigma_e;
  float a, c0, c1, c2; /* update coefficients (signs folded in)                            */
  float w0, w1, w2, w3, w4;
  /* Optional (NULL = off): the launch reads its scalars from DEVICE memory instead of the by-value fields above --
   * 16 floats {a, c0, c1, c2, w0, w1, w2, w3, w4, alpha_e, sigma_e, 5 reserved}, written earlier on the same stream
   * by dpm_adaptive_plan(): the on-device step-size controller of dpm_solver_adaptive (:956-1010), whose next
   * coefficients depend on an accept/reject decision the host never sees. Served by the generic kernel. */
  const float* dev_coef;
} dpm_step_desc;

/* ---- library ------------------------------------------------------------------------ */
DPM_API int dpm_version(void);
DPM_API const char* dpm_last_error(void);

/* Tuning knobs (process-wide, read at launch): variant 0 = direct 128/256-bit global
 * loads, 1 = TMA (cp.async.bulk) shared-memory ring, 2 = auto (default: direct); threads per CTA; CTAs per SM of a
 * persistent grid (0: the direct variant launches one CTA per tile, the ring its built-in shape); 0 keeps the built-in
 * default. Returns DPM_ERR_ARG on invalid values. */
DPM_API int dpm_set_tuning(int variant, int threads, int ctas_per_sm);
DPM_API int dpm_get_tuning(int* variant, int* threads, int* ctas_per_sm);
/* number of kernels launched by this library since load (all streams) */
DPM_API uint64_t dpm_launch_count(void);

/* ---- the general fused step --------------------------------------------------------- */
DPM_API int dpm_step(const dpm_step_desc* desc, dpm_stream_t stream);

/* ---- named entry points, one per reference function --------------------------------- */

/* out = a*x + c0*m0 [+ c1*m1 [+ c2*m2]], k in 1..3. Generic AXPY chain: add_noise :1026,
 * classifier guidance :321, noise_pred_fn conversions :292-298. */
DPM_API int dpm_lincomb(void* out, const void* x, const void* m0, const void* m1, const void* m2,
                int k, float a, float c0, float c1, float c2, uint64_t n, int dtype,
                dpm_stream_t stream);

/* DPM_Solver.dpm_solver_first_update :547-592.  x_t = a*x + c0*model_s
 * (++: a = sigma_t/sigma_s, c0 = -(alpha_t*expm1(-h)); eps: a = exp(dlog_alpha),
 * c0 = -(sigma_t*expm1(h))). */
DPM_API int dpm_solver_first_update(void* x_t, const void* x, const void* model_s, float a, float c0,
                            uint64_t n, int dtype, dpm_stream_t stream);

/* DPM_Solver.multistep_dpm_solver_second_update :796-852.
 * D1_0 = inv_r0*(model_prev_0 - model_prev_1); x_t = a*x + c0*model_prev_0 + c1*D1_0. */
DPM_API int dpm_multistep_second_update(void* x_t, const void* x, const void* model_prev_0,
                                const void* model_prev_1, float a, float c0, float c1,
                                float inv_r0, uint64_t n, int dtype, dpm_stream_t stream);

/* DPM_Solver.multistep_dpm_solver_third_update :854-904.
 * inv_r0 = 1/r0, inv_r1 = 1/r1, w = r0/(r0+r1), q = 1/(r0+r1). */
DPM_API int dpm_multistep_third_update(void* x_t, const void* x, const void* model_prev_0,
                               const void* model_prev_1, const void* model_prev_2, float a,
                               float c0, float c1, float c2, float inv_r0, float inv_r1,
                               float w, float q, uint64_t n, int dtype, dpm_stream_t stream);

/* The difference step shared by singlestep_dpm_solver_second_update :636-669 and
 * singlestep_dpm_solver_third_update :728-739 / :767-778:
 * x_t = a*x + c0*model_s + c1*(model_new - model_s). */
DPM_API int dpm_singlestep_diff_update(void* x_t, const void* x, const void* model_s,
                               const void* model_new, float a, float c0, float c1, uint64_t n,
                               int dtype, dpm_stream_t stream);

/* singlestep_dpm_solver_third_update, solver_type='taylor' :741-750 / :780-789. */
DPM_API int dpm_singlestep_third_taylor_update(void* x_t, const void* x, const void* model_s,
                                       const void* model_s1, const void* model_s2, float a,
                                       float c0, float c1, float c2, float inv_r1, float inv_r2,
                                       float r2, float r1, float r2_minus_r1, uint64_t n,
                                       int dtype, dpm_stream_t stream);

/* model_wrapper.model_fn classifier-free branch :329-330:
 * eps = eps_uncond + scale*(eps_cond - eps_uncond). */
DPM_API int dpm_cfg_combine(void* eps, const void* eps_uncond, const void* eps_cond, float scale,
                    uint64_t n, int dtype, dpm_stream_t stream);

/* model_wrapper.model_fn classifier-free branch :326: x_in = torch.cat([x] * 2). out holds 2*n elements; x is read
 * once and written to out[0, n) and out[n, 2n). (Inside the sampling loop dpm_step's out2 does this for free; this
 * entry serves the first evaluation of a run.) */
DPM_API int dpm_duplicate(void* out, const void* x, uint64_t n, int dtype, dpm_stream_t stream);

/* DPM_Solver.data_prediction_fn :433-442 (without corrector when thr == NULL):
 * x0 = (x - sigma_t*eps)/alpha_t, then optional clamp(x0,-thr_b,thr_b)/thr_b. */
DPM_API int dpm_data_prediction(void* x0, const void* x, const void* eps, float alpha_t, float sigma_t,
                        const float* thr, uint64_t per_sample, uint64_t n, int dtype,
                        dpm_stream_t stream);

/* ---- noise drawn inside the kernel (torch.randn-compatible Philox) ------------------------------------------
 * ATen's launch policy for an fp32 randn of `numel` elements on the current device.
 *   grid: the grid of one launch over all `numel` elements (calc_execution_policy).
 *   counter_offset: the TOTAL amount the caller must advance the torch CUDA generator's philox offset by afterwards.
 *     Up to 2^29 elements that is the one launch's counter offset. Above, ATen splits the tensor into pieces that
 *     fit 32-bit indexing and draws each with its own grid and philox state, so the total is the whole tensor's
 *     counter offset plus each piece's; the kernels below replay the same pieces. */
DPM_API int dpm_philox_policy(uint64_t numel, uint32_t* grid, uint64_t* counter_offset);

/* DPM_Solver.add_noise(x, t, noise=None) :1012-1030 with the noise generated in registers:
 *   xt[i] = alpha_t[i]*x + sigma_t[i]*randn[i],  i < t_count <= 16 (alpha_t, sigma_t: HOST arrays),  xt: [t_count, n].
 * (seed, offset) = the torch CUDA generator's state; for that state the result equals
 * torch.randn((t_count, n)) followed by the reference's three eager ops, bit for bit. x_dtype -> out_dtype: the
 * reference's promotion (16-bit x, fp32 result) or 16-bit storage. */
DPM_API int dpm_add_noise_philox(void* xt, const void* x, uint64_t n, int t_count, const float* alpha_t,
                                 const float* sigma_t, uint64_t seed, uint64_t offset, int x_dtype, int out_dtype,
                                 dpm_stream_t stream);

/* DiffEdit corrector (examples/stable-diffusion/scripts/diffedit_inpaint.ipynb corrector_fn + sampler.py:92-96):
 *   out = x*mask + (1 - mask)*(alpha_t*x0 + sigma_t*randn_like(x0)),  one launch, noise in registers.
 * mask: fp32, mask_n elements, broadcast over the leading dimensions of x (n % mask_n == 0). */
DPM_API int dpm_diffedit_corrector(void* out, const void* x, const void* x0, const float* mask, uint64_t mask_n,
                                   uint64_t n, float alpha_t, float sigma_t, uint64_t seed, uint64_t offset,
                                   int dtype, dpm_stream_t stream);

/* DPM_Solver.dynamic_thresholding_fn :416-423, first half: per-sample
 * s_b = max(quantile(|x0_b|, q), max_val) with torch.quantile's linear interpolation between
 * the two adjacent order statistics (rank arithmetic in fp32). x0 is recomputed on the fly from
 * the same inputs dpm_step() takes (desc->x/xe, e_cond, e_uncond, param, guidance, alpha_e,
 * sigma_e; predict_x0 must be 1); desc->thr/form/out/m* are ignored. Always exact.
 * With a workspace of dpm_dynamic_threshold_workspace() bytes (16-byte aligned device memory,
 * contents irrelevant) samples of >= 8192 elements take the streaming pipeline: pivot sampling,
 * one HBM-rate count/compact pass, exact finish on the ~2 % of keys inside the bracket. Without
 * it (workspace == NULL), or for smaller samples, one thread-block cluster per sample runs a
 * radix select with the keys staged in (distributed) shared memory. s_out: fp32 [n/per_sample]. */
DPM_API size_t dpm_dynamic_threshold_workspace(uint64_t n_samples, uint64_t per_sample);
DPM_API int dpm_dynamic_threshold(float* s_out, const dpm_step_desc* desc, float q, float max_val,
                                  void* workspace, size_t workspace_bytes, dpm_stream_t stream);

/* DPM_Solver.dpm_solver_adaptive error estimate :999-1001:
 *   delta = max(atol, rtol*max(|x_lower|, |x_prev|));
 *   E = max over samples of sqrt(mean(((x_higher - x_lower)/delta)^2))  ->  e_out[0] (device fp32).
 * One streaming pass + a one-CTA epilogue, deterministic reduction order. workspace: device memory
 * of dpm_adaptive_error_workspace(n, per_sample) bytes. */
DPM_API size_t dpm_adaptive_error_workspace(uint64_t n, uint64_t per_sample);
DPM_API int dpm_adaptive_error(float* e_out, const void* x_higher, const void* x_lower,
                               const void* x_prev, float atol, float rtol, uint64_t per_sample,
                               uint64_t n, int dtype, void* workspace, size_t workspace_bytes,
                               dpm_stream_t stream);

/* ---- guidance rescale (Lin et al. 2023, "Common Diffusion Noise Schedules and Sample Steps are Flawed") ------
 * Classifier-free guidance with the guided prediction rescaled toward the standard deviation of the conditional one,
 * in the network's output space (eps for a noise network, v for a v network):
 *   g  = e_uncond + guidance*(e_cond - e_uncond)                       (:330, on the raw outputs)
 *   r_b = fl32(std(e_cond_b)) / fl32(std(g_b))                          (per sample, unbiased, fp64 accumulation)
 *   g' = phi*(g*r_b) + one_minus_phi*g                                  (each op rounded to fp32)
 * then g' takes the place of the combined output in dpm_step (parameterisation :288-298, eps->x0, clamp, update).
 *
 * dpm_cfg_rescale_ratio: r -> ratio_out, fp32 [n/per_sample]. e_cond, e_uncond: n elements of model_dtype each.
 *   One streaming pass with fp64 per-chunk moments and a final kernel that merges them in chunk order: the bits of
 *   r_b depend on sample b's values only. A sample of one element gives NaN (unbiased std), a constant guided sample
 *   inf or NaN; nothing is clamped. workspace: dpm_cfg_rescale_workspace(n/per_sample, per_sample) bytes of 8-byte
 *   aligned device memory (contents irrelevant).
 * dpm_step_rescaled: dpm_step with the rescale; desc->n_model == 2, desc->per_sample set (dividing n),
 *   desc->raw_round == 0. ratio: device fp32 [n/per_sample] (from dpm_cfg_rescale_ratio, same guidance).
 *   phi, one_minus_phi: fl32(phi) and fl32(1 - phi) with 1 - phi formed in double. Served by the direct vector
 *   kernels (tails, unaligned views and dev_coef launches by the generic kernel); never by the TMA variant. */
DPM_API size_t dpm_cfg_rescale_workspace(uint64_t n_samples, uint64_t per_sample);
DPM_API int dpm_cfg_rescale_ratio(float* ratio_out, const void* e_cond, const void* e_uncond, float guidance,
                                  uint64_t per_sample, uint64_t n, int model_dtype,
                                  void* workspace, size_t workspace_bytes, dpm_stream_t stream);
DPM_API int dpm_step_rescaled(const dpm_step_desc* desc, const float* ratio, float phi, float one_minus_phi,
                              dpm_stream_t stream);

/* ---- per-sample classifier-free guidance ------------------------------------------------------------------
 * The scale of the CFG combine (:330) as a device fp32 array guidance[n/per_sample], one value per sample, in place
 * of desc->guidance (ignored by both entries). Sample b with guidance[b] == 1 gets the reference's bypass (:323): the
 * converted conditional output alone, with no combine and no rescale. The values are read on the device only, so a
 * captured graph picks up new values written into the array between replays.
 * dpm_step_guided: dpm_step with the per-sample scale; ratio NULL = plain CFG, else the guidance rescale of
 *   dpm_step_rescaled with that ratio (from dpm_cfg_rescale_ratio_guided) and phi, one_minus_phi.
 *   Needs desc->n_model == 2, desc->raw_round == 0, desc->per_sample != 0 dividing n and a non-NULL guidance;
 *   DPM_ERR_ARG otherwise. Served by the direct vector kernels (tails, unaligned views and dev_coef launches by the
 *   generic kernel); never by the TMA variant.
 * dpm_cfg_rescale_ratio_guided: dpm_cfg_rescale_ratio with g_b = e_uncond + guidance[b]*(e_cond - e_uncond). */
DPM_API int dpm_step_guided(const dpm_step_desc* desc, const float* guidance, const float* ratio, float phi,
                            float one_minus_phi, dpm_stream_t stream);
DPM_API int dpm_cfg_rescale_ratio_guided(float* ratio_out, const void* e_cond, const void* e_uncond,
                                         const float* guidance, uint64_t per_sample, uint64_t n, int model_dtype,
                                         void* workspace, size_t workspace_bytes, dpm_stream_t stream);

/* ---- adaptive projected guidance (Sadat, Hilliges and Weber, ICLR 2025, arXiv:2410.02416) ---------------------
 * Classifier-free guidance on the denoised prediction, with the guidance difference split into a part parallel to the
 * conditional prediction, down-weighted by eta, and a part orthogonal to it; optionally norm-clipped and with reverse
 * momentum across evaluations. Per sample b of per_sample elements, with both outputs first converted to x0 by the
 * parameterisation as a predict_x0 step converts them (alpha_e, sigma_e: the marginals; DPM_PARAM_EDM: its x0 words),
 * every op rounded to fp32:
 *   c = x0(e_cond), u = x0(e_uncond), D = c - u
 *   R = D  (r_prev == NULL)   or   R = D + momentum*r_prev                          (two rounded ops)
 *   k_b = min(1, norm_threshold/||R_b||) if norm_threshold > 0, else 1
 *   p_b = <R_b, c_b> / max(||c_b||, 1e-12)^2
 *   A_b = 1 - (w_b - 1)*(1 - eta)*k_b*p_b,  B_b = (w_b - 1)*k_b                      (fp64, each rounded to fp32 once)
 *   guided = A_b*c + B_b*R      (two products and a sum, each rounded; a sample with guidance[b] == 1: c itself)
 * The sums run over the sample's elements in fp64, per 8192-element chunk, merged in chunk order: the bits of A_b, B_b
 * depend on sample b's values only. w_b = guidance[b] when the per-sample array is given, else desc->guidance.
 * dpm_apg_words: A -> words[0 .. B), B -> words[B .. 2B), B = n/per_sample, fp32 device memory. Reads desc->xe (NULL =>
 *   desc->x), e_cond, e_uncond, param, alpha_e, sigma_e, guidance, dtypes and dev_coef (alpha_e, sigma_e from the
 *   block); form, thr, outputs and predict_x0 are not read. r_out (optional, fp32 [n]) receives R and may be r_prev
 *   (element-wise in place). workspace: dpm_apg_workspace(n/per_sample, per_sample) bytes of 8-byte aligned device
 *   memory (contents irrelevant). Two launches.
 * dpm_step_apg: dpm_step with the guided value in place of the combine: for predict_x0 it is the buffered x0 (the clamp
 *   by thr follows), else eps = (xe - alpha_t*guided)/sigma_t (:292; with dev_coef, alpha_t and sigma_t are read from
 *   the block like alpha_e, sigma_e). r: the R that dpm_apg_words wrote, read in place of e_uncond, or NULL (R = D from
 *   e_uncond). guidance: NULL, or the per-sample scales (only their value 1 is read here).
 * Both need desc->n_model == 2, desc->raw_round == 0, desc->per_sample != 0 dividing n and words != NULL, and refuse
 * DPM_PARAM_EDM with dev_coef and a thr without predict_x0 (DPM_ERR_ARG). dpm_step_apg is served by the direct vector
 * kernels (tails, unaligned views and dev_coef launches by the generic kernel); never by the TMA variant. */
DPM_API size_t dpm_apg_workspace(uint64_t n_samples, uint64_t per_sample);
DPM_API int dpm_apg_words(float* words, const dpm_step_desc* desc, const float* guidance, float eta,
                          float norm_threshold, float momentum, const float* r_prev, float* r_out, void* workspace,
                          size_t workspace_bytes, dpm_stream_t stream);
DPM_API int dpm_step_apg(const dpm_step_desc* desc, const float* words, const float* guidance, const float* r,
                         float alpha_t, float sigma_t, dpm_stream_t stream);

/* ---- CFG-Zero* (Fan, Zheng, Yeh and Liu, "CFG-Zero*: Improved Classifier-Free Guidance for Flow Matching Models",
 * 2025, arXiv:2503.18886) -------------------------------------------------------------------------------------------
 * Classifier-free guidance against the unconditional output scaled per sample by its least-squares fit to the
 * conditional one, in the network's raw output space. Per sample b of per_sample elements (c = e_cond, u = e_uncond,
 * both flattened in storage order):
 *   s*_b = fl32( <c_b, u_b> / (||u_b||^2 + 1e-8) )      (fp64 sums of the fp32-widened outputs, fp64 division)
 *   us = u*s*_b,  g = us + w_b*(c - us)                 (three ops, each rounded to fp32, in this order)
 * and the parameterisation then converts g as it converts a single output (dpm_step with n_model == 1 on g). A sample
 * with w_b == 1 gets the converted c alone. The sums run per 8192-element chunk, merged in chunk order, so the bits of
 * s*_b depend on sample b's values only.
 * dpm_cfgzero_scale: s*_b -> s_out[0 .. n/per_sample), fp32 device memory. Reads the two halves only (2*s_model bytes
 *   per element). workspace: dpm_cfgzero_workspace(n/per_sample, per_sample) bytes of 8-byte aligned device memory
 *   (contents irrelevant). Two launches.
 * dpm_step_cfgzero: dpm_step with g in place of the combine. guidance: NULL (w_b = desc->guidance) or the per-sample
 *   scales, fp32 [n/per_sample] in device memory. Needs desc->n_model == 2, desc->raw_round == 0, desc->per_sample != 0
 *   dividing n and s_star != NULL (DPM_ERR_ARG). Served by the IEEE-division instantiations of the direct vector
 *   kernels for per-sample guidance (tails, unaligned views and dev_coef launches by the generic kernel); never by the
 *   TMA variant. Call the scale pass and then the step on one stream; neither synchronises or allocates. */
DPM_API size_t dpm_cfgzero_workspace(uint64_t n_samples, uint64_t per_sample);
DPM_API int dpm_cfgzero_scale(float* s_out, const void* e_cond, const void* e_uncond, int model_dtype,
                              uint64_t per_sample, uint64_t n, void* workspace, size_t workspace_bytes,
                              dpm_stream_t stream);
DPM_API int dpm_step_cfgzero(const dpm_step_desc* desc, const float* s_star, const float* guidance,
                             dpm_stream_t stream);

/* ---- TCFG ("TCFG: Tangential Damping Classifier-free Guidance", CVPR 2025) ------------------------------------------
 * Classifier-free guidance against the unconditional output projected, per sample, on the first right singular vector
 * v1 of the 2 x per_sample matrix [u; c], in the network's raw output space. Per sample b (c = e_cond, u = e_uncond,
 * both flattened in storage order), A = ||u_b||^2, B = <u_b, c_b>, C = ||c_b||^2 (fp64 sums of the fp32-widened
 * outputs, in the chunking and merge order of dpm_cfgzero_scale), then in fp64 with each op rounded:
 *   h = 0.5*(A - C);  r = sqrt(h*h + B*B)
 *   C >= A:  p = B,  q = (-h) + r;   else:  p = h + r,  q = B
 *   pp = p*p;  n2 = pp + q*q;  wu_b = fl32(pp / n2);  wc_b = fl32((p*q) / n2)
 * so that u' = <u, v1>*v1 = wu_b*u + wc_b*c. n2 == 0 (A == C and B == 0, both outputs zero included) gives (1, 0);
 * a sum that is not finite gives NaN words. Per element, three rounded fp32 ops in this order, then the
 * parameterisation converts g as it converts a single output:
 *   us = u*wu_b + c*wc_b,  g = us + w_b*(c - us)
 * A sample with w_b == 1 gets the converted c alone.
 * dpm_tcfg_words: (wu_b, wc_b) -> w_out[2*b], w_out[2*b + 1] for b < n/per_sample, fp32 device memory. Reads the two
 *   halves only (2*s_model bytes per element). workspace: dpm_tcfg_workspace(n/per_sample, per_sample) bytes of 8-byte
 *   aligned device memory (contents irrelevant). Two launches.
 * dpm_step_tcfg: dpm_step with g in place of the combine. guidance: NULL (w_b = desc->guidance) or the per-sample
 *   scales, fp32 [n/per_sample] in device memory. Needs desc->n_model == 2, desc->raw_round == 0, desc->per_sample != 0
 *   dividing n and words != NULL (DPM_ERR_ARG). Served like dpm_step_cfgzero: the IEEE-division instantiations of the
 *   direct vector kernels for per-sample guidance, the generic kernel for tails, unaligned views and dev_coef
 *   launches, never the TMA variant. Call the words pass and then the step on one stream; neither synchronises or
 *   allocates. Both entry points were added within version 108: test for their symbols. */
DPM_API size_t dpm_tcfg_workspace(uint64_t n_samples, uint64_t per_sample);
DPM_API int dpm_tcfg_words(float* w_out, const void* e_cond, const void* e_uncond, int model_dtype,
                           uint64_t per_sample, uint64_t n, void* workspace, size_t workspace_bytes,
                           dpm_stream_t stream);
DPM_API int dpm_step_tcfg(const dpm_step_desc* desc, const float* words, const float* guidance, dpm_stream_t stream);

/* ---- frequency-decoupled guidance (S. Sadat, T. Vontobel, F. Salehi and R. M. Weber, "Guidance in the Frequency
 * Domain Enables High-Fidelity Sampling at Low CFG Scales", 2025) ----------------------------------------------------
 * Classifier-free guidance with one scale per level of a Laplacian pyramid, in the network's raw output space. Per
 * plane (the last two dims, H x W, of one sample and one index of the other non-batch dims), N = levels scales
 * w_0 (finest) .. w_{N-1} (coarsest), delta_l = fl32(w_l - w_{l-1}), every op fp32, each product rounded, no
 * contraction:
 *   d = c - u;  G_0 = d;  G_{l+1} = Down(G_l)  (l < N-1)
 *   E_{N-1} = delta_{N-1}*G_{N-1};  E_l = delta_l*G_l + Up(E_{l+1})  (l = N-2 .. 1)
 *   g = (u + w_0*d) + Up(E_1)  (N >= 2);  g = u + w_0*d  (N == 1);  stored rounded to model_dtype
 * Filters are 1-D, applied to every row (along W) first, then to every column; R(j) = -j for j < 0, 2(n-1) - j for
 * j > n-1 (reflect without repeating the edge); each term fl(weight*a) with the exact fp32 weights, summed left to right:
 *   Down, n (even) -> n/2:  out[i] = sum_{k=0..5} h_k*a[R(2i-2+k)],  h = [1, 5, 10, 10, 5, 1]/32
 *   Up, m -> 2m:  out[2i]   = (1*a[R(i-2)] + 21*a[R(i-1)] + 35*a[R(i)] + 7*a[R(i+1)])/64
 *                 out[2i+1] = (7*a[R(i-1)] + 35*a[R(i)] + 21*a[R(i+1)] + 1*a[R(i+2)])/64
 * This is the per-level form u_l + w_l*(c_l - u_l) of the Laplacian pyramids of c and u, reconstructed, in exact
 * arithmetic; it needs one pyramid, of d only.
 * dpm_fdg_supported: DPM_OK when a plane of H x W with `levels` levels is served, else DPM_ERR_ARG with the reason in
 *   dpm_last_error(): 1 <= levels <= DPM_FDG_MAX_LEVELS, H and W divisible by 2^(levels-1) with a quotient of at
 *   least 3, H*W <= DPM_FDG_MAX_PLANE. The size rule lives here only.
 * dpm_fdg_guided: g_out <- g for `planes` planes. Plane p is sample s = p / planes_per_sample, index q = p %
 *   planes_per_sample; its element (h, w) is at s*sample_stride + q*plane_stride + h*h_stride + w*w_stride (elements,
 *   the same for g_out, e_cond and e_uncond). scales: scale_stride == 0 -> `levels` shared scales in HOST memory, passed
 *   by value; else per-sample scales in device memory, sample s's at scales[s*scale_stride .. + levels). One launch,
 *   one CTA per plane, every level in shared memory: reads c and u once and writes g once (3*s_model bytes per
 *   element). Dense row-major planes with 16-byte aligned bases take 128-bit accesses; any other strides give the same
 *   bits. Does not synchronise or allocate. */
#define DPM_FDG_MAX_LEVELS 5
#define DPM_FDG_MAX_PLANE 16384   /* H*W: 128 x 128 */
DPM_API int dpm_fdg_supported(uint64_t H, uint64_t W, int levels, int model_dtype);
DPM_API int dpm_fdg_guided(void* g_out, const void* e_cond, const void* e_uncond, int model_dtype, uint64_t planes,
                           uint64_t H, uint64_t W, int64_t sample_stride, int64_t plane_stride, int64_t h_stride,
                           int64_t w_stride, int levels, const float* scales, uint64_t scale_stride,
                           uint64_t planes_per_sample, dpm_stream_t stream);

/* ---- CFG++ (Chung, Kim, Park, Nam and Ye, "CFG++: Manifold-constrained Classifier Free Guidance for Diffusion
 * Models", ICLR 2025, arXiv:2406.08070) -------------------------------------------------------------------------------
 * A DPM-Solver++ update that denoises with the guided data prediction and re-noises with the unconditional noise. Per
 * element, in fp32 with every op rounded (S = desc->state_dtype):
 *   U = round_S(T_u)   T_u: the x0 dpm_step buffers for e_uncond alone (n_model == 1, same param and words)
 *   G = round_S(T_g)   T_g: the x0 dpm_step buffers for the pair (e_cond, e_uncond) with the sample's scale w_b; a
 *                      sample with a per-sample w_b == 1 takes e_cond alone (as dpm_step_guided); desc->guidance is
 *                      always combined, 1 included
 *   LIN1:  out = (a*x + c0*U) + g*(G - U)
 *   DIFF2: out = ((a*x + c0*U) + g*(G - U)) + c1*(w0*(G - m1))      (m1: the previous update's U)
 * m_out (optional) receives U, out2 (optional) a second copy of out. g is alpha_t of the update's end time: in exact
 * arithmetic LIN1 is then alpha_t*G + sigma_t*eps_u (the paper's DDIM) and DIFF2 the 2M CFG++ recurrence; with
 * e_cond == e_uncond, G == U and both are the plain update. guidance: NULL (w_b = desc->guidance) or the per-sample
 * scales, fp32 [n/per_sample] in device memory (then desc->per_sample must divide n). Needs desc->form LIN1 or DIFF2
 * with c0_on_old == 0, n_model == 2, predict_x0 == 1, thr == NULL, raw_round == 0 and dev_coef == NULL (DPM_ERR_ARG).
 * Reads x, e_cond, e_uncond [, m1] and writes out, out2, m_out: 6*s (LIN1) / 7*s (DIFF2) bytes per element with a
 * state and model type of s bytes. Served by packet kernels for the five dtype pairs (tails, unaligned views and
 * per-sample scales over samples that do not hold whole 8-element packets by the generic kernel); never by the TMA
 * variant. */
DPM_API int dpm_step_cfgpp(const dpm_step_desc* desc, float g, const float* guidance, dpm_stream_t stream);

/* ---- SDE-DPM-Solver++ (Lu et al. 2022, arXiv:2211.01095; k-diffusion's DPM++ 2M / 3M SDE) -----------------------------
 * dpm_step with Gaussian noise added to the update, the noise drawn inside the launch:
 *   out = <the LIN1 / DIFF2 / MS3 expression of dpm_step> + cz*z          (fp32, each op rounded, stored as S)
 * z is torch.randn's value for the element: element i (storage order) of `torch.empty(n).normal_(generator=g)` where g
 * holds (seed, offset) -- the normal of ATen's grid-stride Philox4_32_10 kernel (curand_init(seed, idx, offset), one
 * curand_normal4 per 4*G elements, G = 256*grid), split beyond 2^29 elements as ATen splits it (dpm_philox_policy gives
 * the offset the draw consumes, to advance the generator by). With sde->z set, z is read from there instead (fp32 [n],
 * storage order: a draw materialised by torch under CUDA-graph capture) and seed, offset are ignored.
 * The model stage is dpm_step's, with the optional per-sample words of dpm_step_guided (guidance, ratio, phi,
 * one_minus_phi), dpm_step_cfgzero (s_star) and dpm_step_tcfg (tcfg_words), which mean what they mean there (s_star and
 * tcfg_words exclude each other and the ratio; any of them needs n_model == 2 and desc->per_sample dividing n).
 * Needs desc->form LIN1, DIFF2 or MS3 with c0_on_old == 0, raw_round == 0, dev_coef == NULL and sde->offset % 4 == 0
 * (DPM_ERR_ARG before any launch). Reads and writes the bytes dpm_step reads and writes (x, the network outputs or m0,
 * the older buffers; out, out2, m_out) and no noise bytes: one CUDA thread draws 8 Philox blocks, the 32 normals of four
 * 8-element packets. Packets over a tail or a segment boundary, unaligned views and per-sample words over samples that
 * do not hold whole packets take the element path of the same launch. */
typedef struct dpm_sde_desc {
  const float* z;           /* NULL: draw in the launch from (seed, offset) */
  const float* guidance;    /* per-sample scales [n/per_sample] or NULL */
  const float* ratio;       /* guidance rescale ratio [n/per_sample] or NULL */
  const float* s_star;      /* CFG-Zero* scales [n/per_sample] or NULL */
  const float* tcfg_words;  /* TCFG words [n/per_sample][2] or NULL */
  uint64_t seed, offset;
  float cz;
  float phi, one_minus_phi; /* rescale weights (with ratio) */
} dpm_sde_desc;
DPM_API int dpm_step_sde(const dpm_step_desc* desc, const dpm_sde_desc* sde, dpm_stream_t stream);

/* ---- multi-condition classifier-free guidance (composable prompts, Liu et al. 2022) ----------------------------
 * The network runs once on cat([x] * (n_cond + 1)) with the conditions cat([uc, c_1, ..., c_n]) and returns
 * n_cond + 1 blocks: desc->e_uncond (eps_u) and e_conds[0 .. n_cond-1]. Each block is converted by the
 * parameterisation (:288-298), then
 *   eps = eps_u;  eps = eps + scales[k]*(eps_k - eps_u),  k = 0 .. n_cond-1      (each op rounded to fp32)
 * takes the place of the combined output in dpm_step (eps->x0, clamp, update). No scale is bypassed.
 * dpm_step_multi: dpm_step with that combine; desc->n_model == 2, desc->raw_round == 0; desc->e_cond and desc->out2 are
 *   ignored. scales: HOST array of n_cond floats, copied into the launch (capturable). replicas: NULL, or n_cond
 *   device pointers that receive x_t again (blocks 1..n_cond of the next network input; block 0 is `out`). Returns
 *   DPM_ERR_ARG for n_cond outside 2..DPM_MAX_CONDITIONS, raw_round != 0, n_model != 2, or a NULL output, scale array
 *   or replica pointer, before any launch. Served by the packet kernels for the five dtype pairs (tails, unaligned
 *   views, other pairs and dev_coef launches by the generic kernel).
 * dpm_replicate: torch.cat([x] * copies), out holds copies*n elements; x is read once. It serves the first evaluation
 *   of a run (inside the loop dpm_step_multi's replicas do this for free). */
#define DPM_MAX_CONDITIONS 4
DPM_API int dpm_step_multi(const dpm_step_desc* desc, const void* const* e_conds, const float* scales, int n_cond,
                           void* const* replicas, dpm_stream_t stream);
DPM_API int dpm_replicate(void* out, const void* x, uint64_t n, int copies, int dtype, dpm_stream_t stream);

/* ---- regional classifier-free guidance: a weight map per condition (MultiDiffusion-style region composition) -----
 * dpm_step_multi_masked: dpm_step_multi with the scale of condition k multiplied, per element, by a weight map:
 *   eps = eps_u;  w = scales[k]*m_k(i);  eps = eps + w*(eps_k - eps_u),  k = 0 .. n_cond-1   (each op rounded to fp32,
 *                                                                                               none skipped)
 * The weight of global element i (storage order) is maps[k].w[b*sample_stride + (r % period)], b = i / per_sample,
 * r = i - b*per_sample. maps[k].w == NULL means all ones (then w == scales[k] exactly, and the launch computes what
 * dpm_step_multi computes). Three periods are meant: 1 (one weight per sample), the spatial size S of an
 * NCHW-contiguous x (per_sample == C*S: a pixel map shared by the channels), and per_sample (a full element map in x's
 * storage order); sample_stride is 0 (one map shared by the batch) or period. maps: HOST array of n_cond entries; the
 * weights are fp32 in device memory, read at launch time (a captured graph sees values written into them).
 * Needs 1 <= n_cond <= DPM_MAX_CONDITIONS, desc->per_sample != 0 dividing n, and period != 0 dividing per_sample;
 * otherwise as dpm_step_multi (DPM_ERR_ARG before any launch). The packet kernels serve the five dtype pairs when
 * samples hold whole packets and every map has period 1, or period % 8 == 0 with 16-byte-aligned weights; tails,
 * unaligned views, other maps and pairs and dev_coef launches run on the generic kernel. */
typedef struct dpm_cond_map {
  const float* w;
  uint64_t period;
  uint64_t sample_stride;
} dpm_cond_map;
DPM_API int dpm_step_multi_masked(const dpm_step_desc* desc, const void* const* e_conds, const float* scales,
                                  const dpm_cond_map* maps, int n_cond, void* const* replicas, dpm_stream_t stream);

/* ---- Perp-Neg: perpendicular negative prompts (Armandpour, Sadeghian, Zheng, Sadeghian and Zhou, "Re-imagine the
 * Negative Prompt Algorithm: Transform 2D Diffusion into 3D, alleviate Janus problem and Beyond", arXiv:2304.04968) --
 * Multi-condition guidance in which every condition after the first loses, per sample, its component along the first
 * condition's direction before it is weighted. With u = e_uncond, e_k = e_conds[k-1] (raw network outputs, all K
 * blocks flattened per sample in storage order), in exact arithmetic:
 *   eps = u + s_1*d_1 + sum_{k>=2} s_k*(d_k - (<d_k, d_1>/||d_1||^2)*d_1),   d_k = e_k - u
 * which is u + w_1*d_1 + sum_{k>=2} s_k*d_k with one per-sample weight w_1. Every parameterisation maps the blocks of
 * a sample by one affine map whose x term is shared, so the ratio is the same in raw and converted space.
 * dpm_perpneg_words: w_1 of each sample b -> w_out[b], b < n/per_sample, fp32 device memory. Per sample, each value
 *   widened to fp64 and d_k = e_k - u formed in fp64, the fp64 sums N = sum d_1*d_1 and P_k = sum d_k*d_1 (k = 2..K)
 *   run in the chunking, thread ownership and merge order of dpm_cfgzero_scale, so the word of sample b depends on
 *   sample b's values only. Then c_k = P_k / N (c_k = 0 when N == 0: condition 1 equals u, nothing to project out)
 *   and, in fp64 left to right with each op rounded, sigma_k = fl32(s_k) = scales[k-1] widened:
 *     w_1 = fl32(sigma_1 - sigma_2*c_2 - ... - sigma_K*c_K)
 *   A non-finite N or P_k gives the NaN 0x7fffffff. scales: HOST array of n_cond floats, passed by value (capturable).
 *   Reads the K+1 blocks once ((K+1)*s_model bytes per element). workspace: dpm_perpneg_workspace(n/per_sample,
 *   per_sample) bytes of 8-byte aligned device memory (contents irrelevant). Two launches; does not synchronise or
 *   allocate. Returns DPM_ERR_ARG before any launch for n_cond outside 2..DPM_MAX_CONDITIONS, a NULL pointer (w_out,
 *   e_uncond, e_conds, an entry of it, scales), a bad model_dtype, or per_sample not dividing n. 16-byte aligned blocks
 *   (32-byte for fp32) with per_sample % 8 == 0 take 128-bit loads; anything else gives the same bits element-wise.
 * The step is then dpm_step_multi_masked with scales (1, s_2, .., s_K), maps[0] = {w_out, 1, 1} and no other map:
 *   eps_u + w_1*(eps_1 - eps_u) + s_2*(eps_2 - eps_u) + ..., each block converted by the parameterisation first (1*w_1
 *   is w_1 exactly). Both entry points were added within version 108: test for their symbols. */
DPM_API size_t dpm_perpneg_workspace(uint64_t n_samples, uint64_t per_sample);
DPM_API int dpm_perpneg_words(float* w_out, const void* e_uncond, const void* const* e_conds, const float* scales,
                              int n_cond, int model_dtype, uint64_t per_sample, uint64_t n, void* workspace,
                              size_t workspace_bytes, dpm_stream_t stream);

/* ---- UniPC multistep (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework", arXiv:2302.04867) ------
 * One launch per network evaluation i: the corrector of step i and the predictor of step i+1 (dpm_solver_b200/unipc.py
 * states the method and how the host folds the words below). With x~ = desc->x, the predictor output x~_i that the
 * network was evaluated at, and m_i its model value (desc->n_model >= 1: converted from the raw outputs exactly as
 * dpm_step converts them -- parameterisation, CFG, eps -> x0, clamp -- rounded to the state dtype and written to
 * desc->m_out when set; n_model == 0: read from desc->m0), m_{i-1} = desc->m1, m_{i-2} = desc->m2, m_{i-3} = u->m3:
 *   pc > 0 : x_i = x~ [+ cd[0]*(m_{i-2} - m_{i-1}) [+ cd[1]*(m_{i-3} - m_{i-1})]] + ct*(m_i - m_{i-1})
 *            (cd[0] from pc >= 2, cd[1] from pc == 3), rounded to the state dtype in registers
 *   pc = 0 : x_i = x~
 *   pp > 0 : x~_{i+1} = a*x_i + c0*m_i [+ cp[0]*(m_{i-1} - m_i) [+ cp[1]*(m_{i-2} - m_i)]]  (cp[0] from pp >= 2,
 *            cp[1] from pp == 3) -> desc->out, and desc->out2 when set (the doubled CFG batch)
 *   out_c  : optional, receives x_i (intermediates, hooks); required when pp == 0
 * Differences first, then the sums left to right, each product and sum rounded to fp32. desc->xe, form, c0_on_old
 * and a, c0..c2, w0..w4 are not read. Returns DPM_ERR_ARG before any launch for pc or pp outside 0..3, pc == pp == 0,
 * raw_round != 0, dev_coef != NULL, or a NULL operand the orders need. Served by packet kernels for the five dtype
 * pairs (tails, unaligned views and other pairs by the generic kernel); never by the TMA variant. */
typedef struct dpm_unipc_desc {
  const void* m3;   /* m_{i-3}, state dtype; read when pc == 3 */
  void* out_c;      /* optional: the corrected state x_i      */
  int32_t pc;       /* corrector order 0..3 (0 = off)         */
  int32_t pp;       /* predictor order 0..3 (0 = none)        */
  float cd[2], ct;  /* corrector words                        */
  float a, c0;      /* predictor words                        */
  float cp[2];
} dpm_unipc_desc;
DPM_API int dpm_step_unipc(const dpm_step_desc* desc, const dpm_unipc_desc* u, dpm_stream_t stream);

/* ---- dpm_solver_adaptive with the controller on the device (:956-1010) -------------------------------------
 * Device buffers (caller-allocated, fp32): state[16] (s, lambda_s, lambda_0, h, t, nfe, done, accept, iterations as
 * int bit patterns where integral), coef[4][16] (one dpm_step_desc.dev_coef block per fused launch of an
 * iteration), times[6] (evaluation times s, s1, s2, then the model-input times the network receives), error[1]
 * (written by dpm_adaptive_error). Schedule: discrete (tables as NoiseScheduleVP holds them, plus their flipped
 * copies, all on the device), the continuous linear VPSDE, or the flow schedule (NoiseScheduleFlow's closed forms:
 * sigma_t = shift*t/(1 + (shift-1)*t), alpha_t = 1 - sigma_t; the network then receives time_scale*sigma_t).
 *   dpm_adaptive_init   : s = t_T, lambda_s, lambda_0, h = h_init                                      :972-977
 *   dpm_adaptive_plan   : t = lambda^-1(lambda_s + h) and every coefficient block / time label of the
 *                         lower- and higher-order updates of this iteration                             :984-992
 *   dpm_adaptive_decide : E <= 1 ? accept (s = t, lambda_s) ; h = min(theta*h*E^(-1/order), lambda_0 - lambda_s);
 *                         nfe += order; done = |s - t_0| <= t_err (2 = NaN error estimate)              :1002-1008
 *   dpm_select_copy     : dst <- src iff the last decide accepted (x <- x_higher, x_prev <- x_lower)     :1003-1005
 * Launch order per iteration for order 2: plan, [net(x,s)] step(coef 0: x_lower), step(coef 1: x_s1, pure),
 * [net(x_s1,s1)] step(coef 2: x_higher), error, decide, select_copy x2; order 3 uses coef 0..3 (see
 * dpm_solver_b200/solver.py). After `done` the plan emits identity coefficients, so a fixed-length chunk of
 * iterations can be enqueued (or graph-captured) and `done` read back once per chunk. */
typedef struct dpm_adaptive_ctl {
  int32_t schedule_kind;       /* 0 discrete, 1 linear, 2 flow */
  int32_t table_len;
  const float* t_array;        /* device, [table_len] */
  const float* log_alpha_array;
  const float* log_alpha_flipped;
  const float* t_flipped;
  float beta_0, beta_1_minus_beta_0, inv_total_N;
  int32_t discrete_time_input; /* 1: the network takes (t - 1/N)*1000 (:278), 0: t */
  int32_t order;               /* 2 or 3 */
  int32_t predict_x0;          /* dpmsolver++ */
  int32_t taylor;              /* solver_type == 'taylor' */
  float t_0, theta, t_err;
  float* state;                /* device [16] */
  float* coef;                 /* device [4][16] */
  float* times;                /* device [6] */
  const float* error;          /* device [1] */
  float beta_0_sq;             /* linear: fl32(beta_0**2) with the square taken in double (reference :162) */
  float flow_shift;            /* flow: fl32(shift) */
  float flow_shift_minus_1;    /* flow: fl32(shift - 1), the difference taken in double */
  float flow_time_scale;       /* flow: the network takes fl32(time_scale)*sigma_t (discrete_time_input is not read) */
} dpm_adaptive_ctl;

DPM_API int dpm_adaptive_init(const dpm_adaptive_ctl* ctl, float t_T, float h_init, dpm_stream_t stream);
DPM_API int dpm_adaptive_plan(const dpm_adaptive_ctl* ctl, dpm_stream_t stream);
DPM_API int dpm_adaptive_decide(const dpm_adaptive_ctl* ctl, dpm_stream_t stream);
DPM_API int dpm_select_copy(void* dst, const void* src, const float* state, uint64_t bytes, dpm_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DPM_SOLVER_B200_H */
