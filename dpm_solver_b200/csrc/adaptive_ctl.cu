// adaptive_ctl.cu -- the step-size controller of dpm_solver_adaptive ON THE DEVICE (dpm_solver_pytorch.py:956-1010).
//
// The reference decides on the host every iteration (`torch.all(E <= 1.)` :1002 syncs, and every schedule scalar
// of the next step depends on the decision). Here the controller state (s, lambda_s, h, nfe, done) lives in device
// memory and three tiny kernels bracket the heavy ones of an iteration:
//
//   k_adapt_plan   (1 thread) : t = lambda^-1(lambda_s + h) :984, the marginals of s, s1, s2, t and the coefficient
//                               block of every launch of the lower- and higher-order updates (the formulas of
//                               plan.py, i.e. :563-588, :613-669, :697-789, same fp32 op order; device libm), the time
//                               labels and model-input times the network receives
//   ... model evaluations + fused step launches that READ their scalars from those blocks (dpm_step_desc.dev_coef),
//       then the error estimate (adaptive.cu) ...
//   k_adapt_decide (1 thread) : accept = E <= 1 :1002; s, lambda_s :1003-1006; h = min(theta*h*E^(-1/order),
//                               lambda_0 - lambda_s) :1007; nfe += order :1008; done = |s - t_0| <= t_err :983
//   k_select_copy             : x <- x_higher, x_prev <- x_lower when accepted (:1003-1005), a no-op otherwise
//
// The host enqueues a fixed-length chunk of iterations and reads `done`/`nfe` back once per chunk. After `done`
// the plan kernel emits identity coefficients at t_0, so the surplus iterations of a chunk leave x untouched.
//
// Contract: the reference's fp32 operation order (plan.py / schedule.py and the host controller's update), with
// exp/log/expm1/log1p evaluated in fp64 and rounded once -- correctly rounded fp32 -- and float_power(E, -1/order)
// rounded to fp64 and then to fp32 as the reference does. tests/adaptive_oracle.py evaluates exactly that (mpmath
// for the transcendentals) and tests/test_gpu_adaptive_controller.py requires every word these kernels write to be
// bit-identical to it; only where the exact value lies within the fp64 libm's error (1 ulp, 2 for pow) of an fp32
// rounding boundary is either neighbour accepted. The host's fp32 libm differs in the last ulp of some arguments,
// so end to end the sample agrees with the reference to the north-star tolerance and the accept/reject sequence --
// hence NFE -- is identical unless E lands within ~1e-6 of 1 (tests/test_adaptive.py).
#include <math.h>

#include "common.cuh"
#include "launch.cuh"

namespace dpm {

// device view of NoiseScheduleVP
struct SchedDev {
  int32_t kind;            // 0 discrete (tables), 1 linear
  int32_t K;               // table length
  const float* t;          // [K] ascending
  const float* la;         // [K] log alpha (descending in value)
  const float* la_f;       // [K] flipped log alpha (ascending)
  const float* t_f;        // [K] flipped t
  float beta_0, beta_d;    // linear: beta_0, fl(beta_1 - beta_0)
  float beta_0_sq;         // linear: fl(beta_0**2), squared in double like the reference's python float (:162)
  float inv_N;             // fl(1 / total_N) (model-input time of discrete-time networks :278)
  int32_t discrete_input;  // 1: network takes (t - 1/N)*1000, 0: t itself
};

struct AdaptCfg {
  SchedDev ns;
  int32_t order;           // 2: DPM-Solver-12, 3: DPM-Solver-23
  int32_t pp;              // 1: dpmsolver++ (data prediction), 0: dpmsolver
  int32_t taylor;          // solver_type == 'taylor'
  float t_0, theta, t_err;
  float* state;            // AdaptState (device)
  float* coef;             // [kLaunches][kCoefWords] coefficient blocks (device)
  float* times;            // [3] evaluation times s, s1, s2; [3..5] model-input times
  const float* E;          // error estimate of this iteration (device, written by k_err_final)
};

enum { ST_S = 0, ST_LAM_S = 1, ST_LAM_0 = 2, ST_H = 3, ST_T = 4, ST_NFE = 5, ST_DONE = 6, ST_ACCEPT = 7, ST_ITERS = 8, ST_WORDS = 16 };

// Transcendentals: evaluated in fp64 and rounded once, i.e. correctly rounded fp32 results. The host's (SLEEF) fp32
// functions are within one ulp of that, and these formulas amplify an ulp (phi_3 = phi_2/h - 0.5 cancels), so the
// closer the scalars the closer the adaptive path follows the reference's; one thread runs this, fp64 costs nothing.
__device__ __forceinline__ float exp_cr(float v) { return (float)exp((double)v); }
__device__ __forceinline__ float log_cr(float v) { return (float)log((double)v); }
__device__ __forceinline__ float expm1_cr(float v) { return (float)expm1((double)v); }
__device__ __forceinline__ float log1p_cr(float v) { return (float)log1p((double)v); }

// y(x) on ascending keypoints, linear extrapolation, the reference's bracket rule (schedule.py _piecewise_linear)
__device__ float interp(const float* xp, const float* yp, int K, float x) {
  int lo = 0, hi = K;                      // i = #{xp < x}
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (xp[mid] < x) lo = mid + 1; else hi = mid;
  }
  int j0 = lo - 1;
  j0 = j0 < 0 ? 0 : (j0 > K - 2 ? K - 2 : j0);
  const float x0 = xp[j0], x1 = xp[j0 + 1], y0 = yp[j0], y1 = yp[j0 + 1];
  return y0 + (x - x0) * (y1 - y0) / (x1 - x0);   // :1291
}
__device__ float logaddexp0(float v) {     // logaddexp(0, v) as ATen computes it: max + log1p(exp(-|a - b|))
  const float m = fmaxf(0.f, v);
  return m + log1p_cr(exp_cr(-fabsf(v)));
}
__device__ float log_alpha_of(const SchedDev& ns, float t) {
  if (ns.kind == 0) return interp(ns.t, ns.la, ns.K, t);                       // :129
  return -0.25f * (t * t) * ns.beta_d - 0.5f * t * ns.beta_0;                  // :134
}
__device__ float inverse_lambda(const SchedDev& ns, float lamb) {
  if (ns.kind == 1) {                                                            // :161-163
    const float tmp = (2.f * ns.beta_d) * logaddexp0(-2.f * lamb);
    const float Delta = ns.beta_0_sq + tmp;
    return tmp / (sqrtf(Delta) + ns.beta_0) / ns.beta_d;
  }
  const float la = -0.5f * logaddexp0(-2.f * lamb);                             // :165
  return interp(ns.la_f, ns.t_f, ns.K, la);                                     // :166
}
struct Marg { float t, la, sigma, lam, alpha; };
__device__ Marg marg(const SchedDev& ns, float t) {
  Marg m;
  m.t = t;
  m.la = log_alpha_of(ns, t);
  const float e2 = 1.f - exp_cr(2.f * m.la);
  m.sigma = sqrtf(e2);                    // :146
  m.lam = m.la - 0.5f * log_cr(e2);         // :153-154
  m.alpha = exp_cr(m.la);                   // :140
  return m;
}

// one coefficient block (dpm_step_desc.dev_coef): the scalars of one fused launch
enum { CO_A = 0, CO_C0, CO_C1, CO_C2, CO_W0, CO_W1, CO_W2, CO_W3, CO_W4, CO_ALPHA_E, CO_SIGMA_E, CO_WORDS = 16 };
__device__ void put(float* b, float a, float c0, float c1, float c2, float w0, float w1, float w2, float w3, float w4,
                    float alpha_e, float sigma_e) {
  b[CO_A] = a; b[CO_C0] = c0; b[CO_C1] = c1; b[CO_C2] = c2; b[CO_W0] = w0; b[CO_W1] = w1; b[CO_W2] = w2;
  b[CO_W3] = w3; b[CO_W4] = w4; b[CO_ALPHA_E] = alpha_e; b[CO_SIGMA_E] = sigma_e;
}
// dpm_solver_first_update :563-588
__device__ void first_update(bool pp, const Marg& ms, const Marg& mt, float& a, float& c0) {
  const float h = mt.lam - ms.lam;
  if (pp) { a = mt.sigma / ms.sigma; c0 = -(mt.alpha * expm1_cr(-h)); }
  else { a = exp_cr(mt.la - ms.la); c0 = -(mt.sigma * expm1_cr(h)); }
}

__global__ void k_adapt_plan(const AdaptCfg c) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float* st = c.state;
  float* co = c.coef;
  const bool pp = c.pp != 0;
  if (__float_as_int(st[ST_DONE]) != 0) {
    // finished: identity updates at t_0 for the rest of the chunk (x_lower = x_higher = x)
    const Marg m0 = marg(c.ns, c.t_0);
    for (int l = 0; l < 4; ++l) put(co + l * CO_WORDS, 1.f, 0.f, 0.f, 0.f, 1.f, 1.f, 1.f, 1.f, 1.f, m0.alpha, m0.sigma);
    for (int j = 0; j < 3; ++j) {
      c.times[j] = c.t_0;
      c.times[3 + j] = c.ns.discrete_input ? (c.t_0 - c.ns.inv_N) * 1000.f : c.t_0;
    }
    return;
  }
  const float s = st[ST_S], lam_s = st[ST_LAM_S], hstep = st[ST_H];
  const float t = inverse_lambda(c.ns, lam_s + hstep);                          // :984
  st[ST_T] = t;
  const Marg ms = marg(c.ns, s), mt = marg(c.ns, t);
  const float h = mt.lam - ms.lam;
  float tt[3] = {s, s, s};
  if (c.order == 2) {
    // lower: first update s -> t (launch 0, consumes the evaluation at s)
    float a, c0;
    first_update(pp, ms, mt, a, c0);
    put(co + 0 * CO_WORDS, a, c0, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, ms.alpha, ms.sigma);
    // higher: singlestep second update, r1 = 0.5 (:613-669): launch 1 = x -> x_s1 (pure), launch 2 = final
    const float r1 = 0.5f;
    const float s1 = inverse_lambda(c.ns, ms.lam + r1 * h);
    const Marg m1 = marg(c.ns, s1);
    tt[1] = s1;
    float a1, c01, af, bf, c1f;
    if (pp) {
      a1 = m1.sigma / ms.sigma; c01 = -(m1.alpha * expm1_cr(-r1 * h));
      const float phi_1 = expm1_cr(-h);
      af = mt.sigma / ms.sigma; bf = mt.alpha * phi_1;
      c1f = c.taylor ? (1.f / r1) * (mt.alpha * (phi_1 / h + 1.f)) : -((0.5f / r1) * bf);
    } else {
      a1 = exp_cr(m1.la - ms.la); c01 = -(m1.sigma * expm1_cr(r1 * h));
      const float phi_1 = expm1_cr(h);
      af = exp_cr(mt.la - ms.la); bf = mt.sigma * phi_1;
      c1f = c.taylor ? -((1.f / r1) * (mt.sigma * (phi_1 / h - 1.f))) : -((0.5f / r1) * bf);
    }
    put(co + 1 * CO_WORDS, a1, c01, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, ms.alpha, ms.sigma);
    put(co + 2 * CO_WORDS, af, -bf, c1f, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, m1.alpha, m1.sigma);
  } else {
    // lower: singlestep second update with r1 = 1/3; higher: singlestep third update r1 = 1/3, r2 = 2/3 (:697-789)
    const float r1 = (float)(1.0 / 3.0), r2 = (float)(2.0 / 3.0);
    const float s1 = inverse_lambda(c.ns, ms.lam + r1 * h), s2 = inverse_lambda(c.ns, ms.lam + r2 * h);
    const Marg m1 = marg(c.ns, s1), m2 = marg(c.ns, s2);
    tt[1] = s1; tt[2] = s2;
    float a1, c01, at, bt, c1low, a2, c02, c12, c1fin, c2fin = 0.f, c1tay = 0.f;
    if (pp) {
      const float phi_11 = expm1_cr(-r1 * h), phi_12 = expm1_cr(-r2 * h), phi_1 = expm1_cr(-h);
      const float phi_22 = expm1_cr(-r2 * h) / (r2 * h) + 1.f, phi_2 = phi_1 / h + 1.f, phi_3 = phi_2 / h - 0.5f;
      a1 = m1.sigma / ms.sigma; c01 = -(m1.alpha * phi_11);
      at = mt.sigma / ms.sigma; bt = mt.alpha * phi_1;
      c1low = c.taylor ? (1.f / r1) * (mt.alpha * (phi_1 / h + 1.f)) : -((0.5f / r1) * bt);
      a2 = m2.sigma / ms.sigma; c02 = -(m2.alpha * phi_12); c12 = r2 / r1 * (m2.alpha * phi_22);
      c1fin = (1.f / r2) * (mt.alpha * phi_2);
      c1tay = mt.alpha * phi_2; c2fin = -(mt.alpha * phi_3);
    } else {
      const float phi_11 = expm1_cr(r1 * h), phi_12 = expm1_cr(r2 * h), phi_1 = expm1_cr(h);
      const float phi_22 = expm1_cr(r2 * h) / (r2 * h) - 1.f, phi_2 = phi_1 / h - 1.f, phi_3 = phi_2 / h - 0.5f;
      a1 = exp_cr(m1.la - ms.la); c01 = -(m1.sigma * phi_11);
      at = exp_cr(mt.la - ms.la); bt = mt.sigma * phi_1;
      c1low = c.taylor ? -((1.f / r1) * (mt.sigma * (phi_1 / h - 1.f))) : -((0.5f / r1) * bt);
      a2 = exp_cr(m2.la - ms.la); c02 = -(m2.sigma * phi_12); c12 = -(r2 / r1 * (m2.sigma * phi_22));
      c1fin = -((1.f / r2) * (mt.sigma * phi_2));
      c1tay = -(mt.sigma * phi_2); c2fin = -(mt.sigma * phi_3);
    }
    put(co + 0 * CO_WORDS, a1, c01, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, ms.alpha, ms.sigma);              // eval s: x -> x_s1
    put(co + 1 * CO_WORDS, at, -bt, c1low, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, m1.alpha, m1.sigma);            // eval s1: lower final
    put(co + 2 * CO_WORDS, a2, c02, c12, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, m1.alpha, m1.sigma);              // pure: x -> x_s2
    if (c.taylor) put(co + 3 * CO_WORDS, at, -bt, c1tay, c2fin, 1.f / r1, 1.f / r2, r2, r1, r2 - r1, m2.alpha, m2.sigma);
    else put(co + 3 * CO_WORDS, at, -bt, c1fin, 0.f, 1.f, 0.f, 0.f, 0.f, 0.f, m2.alpha, m2.sigma);       // eval s2: higher final
  }
  for (int j = 0; j < 3; ++j) {
    c.times[j] = tt[j];
    c.times[3 + j] = c.ns.discrete_input ? (tt[j] - c.ns.inv_N) * 1000.f : tt[j];   // get_model_input_time :278
  }
}

__global__ void k_adapt_decide(const AdaptCfg c) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float* st = c.state;
  st[ST_ACCEPT] = __int_as_float(0);
  if (__float_as_int(st[ST_DONE]) != 0) return;
  st[ST_ITERS] = __int_as_float(__float_as_int(st[ST_ITERS]) + 1);
  const float E = c.E[0];
  if (E != E) { st[ST_DONE] = __int_as_float(2); return; }         // NaN error estimate: stop, the host raises
  if (E <= 1.f) {                                                  // :1002-1006
    st[ST_ACCEPT] = __int_as_float(1);
    st[ST_S] = st[ST_T];
    st[ST_LAM_S] = marg(c.ns, st[ST_T]).lam;
  }
  // h = min(theta * h * float_power(E, -1/order).float(), lambda_0 - lambda_s)   :1007
  // torch.min propagates NaN (E = 0 with h = 0 gives 0 * inf): fminf would drop it and jump to lambda_0 - lambda_s
  const float grow = (float)pow((double)E, -1.0 / (double)c.order);
  const float h = min_nan((c.theta * st[ST_H]) * grow, st[ST_LAM_0] - st[ST_LAM_S]);
  st[ST_H] = h;
  st[ST_NFE] = __int_as_float(__float_as_int(st[ST_NFE]) + c.order);           // :1008
  if (h != h) st[ST_DONE] = __int_as_float(2);   // NaN step: every later estimate is NaN, stop now, the host raises
  if (fabsf(st[ST_S] - c.t_0) <= c.t_err) st[ST_DONE] = __int_as_float(1);     // while |s - t_0| > t_err :983
}

__global__ void k_adapt_init(const AdaptCfg c, float t_T, float h_init) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float* st = c.state;
  for (int i = 0; i < ST_WORDS; ++i) st[i] = 0.f;
  st[ST_S] = t_T;
  st[ST_LAM_S] = marg(c.ns, t_T).lam;         // :974
  st[ST_LAM_0] = marg(c.ns, c.t_0).lam;       // :975
  st[ST_H] = h_init;                          // :976
  if (fabsf(t_T - c.t_0) <= c.t_err) st[ST_DONE] = __int_as_float(1);
}

// dst <- src when *flag != 0 (the accepted step's x_higher / x_lower), else nothing
__global__ void __launch_bounds__(256) k_select_copy(uint4* __restrict__ dst, const uint4* __restrict__ src,
                                                     const float* __restrict__ state, uint64_t n16, char* dtail,
                                                     const char* stail, uint32_t tail) {
  if (__float_as_int(state[ST_ACCEPT]) == 0) return;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (uint64_t)gridDim.x * blockDim.x)
    dst[i] = src[i];
  if (blockIdx.x == 0 && threadIdx.x < tail) dtail[threadIdx.x] = stail[threadIdx.x];
}

static int fill_cfg(AdaptCfg* c, const dpm_adaptive_ctl* a) {
  if (a == nullptr || a->state == nullptr || a->coef == nullptr || a->times == nullptr) { set_error("adaptive controller: NULL buffer"); return DPM_ERR_ARG; }
  if (a->order != 2 && a->order != 3) { set_error("adaptive controller: order must be 2 or 3"); return DPM_ERR_ARG; }
  if (a->schedule_kind == 0 && (a->table_len < 2 || !a->t_array || !a->log_alpha_array || !a->log_alpha_flipped || !a->t_flipped)) {
    set_error("adaptive controller: discrete schedule needs its four tables"); return DPM_ERR_ARG;
  }
  if (a->schedule_kind != 0 && a->schedule_kind != 1) { set_error("adaptive controller: schedule must be discrete (0) or linear (1)"); return DPM_ERR_UNSUPPORTED; }
  memset(c, 0, sizeof(*c));
  c->ns.kind = a->schedule_kind; c->ns.K = a->table_len;
  c->ns.t = a->t_array; c->ns.la = a->log_alpha_array; c->ns.la_f = a->log_alpha_flipped; c->ns.t_f = a->t_flipped;
  c->ns.beta_0 = a->beta_0; c->ns.beta_d = a->beta_1_minus_beta_0; c->ns.beta_0_sq = a->beta_0_sq;
  c->ns.inv_N = a->inv_total_N;
  c->ns.discrete_input = a->discrete_time_input;
  c->order = a->order; c->pp = a->predict_x0; c->taylor = a->taylor;
  c->t_0 = a->t_0; c->theta = a->theta; c->t_err = a->t_err;
  c->state = a->state; c->coef = a->coef; c->times = a->times; c->E = a->error;
  return DPM_OK;
}

int launch_adaptive_init(const dpm_adaptive_ctl* a, float t_T, float h_init, cudaStream_t stream) {
  AdaptCfg c;
  int rc = fill_cfg(&c, a);
  if (rc != DPM_OK) return rc;
  k_adapt_init<<<1, 32, 0, stream>>>(c, t_T, h_init);
  count_launch();
  return DPM_OK;
}
int launch_adaptive_plan(const dpm_adaptive_ctl* a, cudaStream_t stream) {
  AdaptCfg c;
  int rc = fill_cfg(&c, a);
  if (rc != DPM_OK) return rc;
  k_adapt_plan<<<1, 32, 0, stream>>>(c);
  count_launch();
  return DPM_OK;
}
int launch_adaptive_decide(const dpm_adaptive_ctl* a, cudaStream_t stream) {
  AdaptCfg c;
  int rc = fill_cfg(&c, a);
  if (rc != DPM_OK) return rc;
  if (a->error == nullptr) { set_error("adaptive controller: NULL error estimate"); return DPM_ERR_ARG; }
  k_adapt_decide<<<1, 32, 0, stream>>>(c);
  count_launch();
  return DPM_OK;
}
int launch_select_copy(void* dst, const void* src, const float* state, uint64_t bytes, cudaStream_t stream) {
  if (bytes == 0) return DPM_OK;
  if (((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src)) & 15) != 0) { set_error("select copy: 16-byte aligned tensors"); return DPM_ERR_ARG; }
  const uint64_t n16 = bytes / 16;
  const uint32_t tail = (uint32_t)(bytes % 16);
  uint64_t blocks = (n16 + 255) / 256;
  const uint64_t cap = (uint64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks == 0) blocks = 1;
  k_select_copy<<<(unsigned)blocks, 256, 0, stream>>>(static_cast<uint4*>(dst), static_cast<const uint4*>(src), state, n16,
                                                     static_cast<char*>(dst) + n16 * 16, static_cast<const char*>(src) + n16 * 16, tail);
  count_launch();
  return DPM_OK;
}

}  // namespace dpm
