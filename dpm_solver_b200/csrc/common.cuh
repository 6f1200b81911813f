// common.cuh -- shared device code for the DPM-Solver step kernels (sm_90a).
//
// The per-element arithmetic below restates, in fp32 registers, the expression trees of the
// reference dpm_solver_pytorch.py (line numbers cited inline). The translation unit is
// compiled with -fmad=false: every product and every sum is rounded separately, exactly as the
// reference's chain of eager elementwise ops does, so fp32 results are bit-identical.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "dpm_solver_b200.h"

namespace dpm {

constexpr int kPacket = 8;  // elements per thread-packet: 32 B of fp32 (2 x LDG.128) / 16 B of 16-bit

// ---- kernel parameter block (passed by value, __grid_constant__) -------------------------
struct KParams {
  const void* x;
  const void* xe;
  const void* m0;
  const void* m1;
  const void* m2;
  const void* ec;
  const void* eu;
  void* m_out;
  void* out;
  void* out2;
  const float* thr;
  uint64_t n;           // elements (scalar kernel) / unused by packet kernels
  uint32_t npk;         // number of full packets
  uint32_t pk_per_sample;  // per_sample / 8 when per_sample % 8 == 0, else 0
  uint64_t per_sample;
  uint64_t elem_offset;  // global index of element 0 (tail launches), for thr lookup
  int32_t param;
  int32_t predict_x0;
  int32_t c0_on_old;
  int32_t use_xe;    // conversion reads the evaluation state
  int32_t xe_is_x;   // ... and it is the same tensor as x (load once)
  int32_t form;      // runtime copies (scalar kernel only)
  int32_t n_model;
  int32_t state_dtype;
  int32_t model_dtype;
  float guidance, alpha_e, sigma_e;
  float a, c0, c1, c2;
  float w0, w1, w2, w3, w4;
  // correctly rounded reciprocals of the kernel-constant divisors (host computed) and a flag telling
  // the device that the reciprocal-refinement division below is valid for all three of them
  float r_alpha;
  // reference-rounding mode (dpm_step_desc.raw_round): bits 0-1 = 16-bit dtype code the raw network
  // outputs arrived in, bit 2 = buffer differences are taken in that type too. 0 = off. Only the
  // <RND = true> instantiations below read it.
  int32_t raw_round;
  float r_w4;
  int32_t fast_div;
  const float* dev_coef;   // optional: scalars read from device memory (dpm_step_desc.dev_coef); generic kernel only
  // guidance rescale (dpm_step_rescaled): per-sample ratio std(out_c)/std(g), fp32 [n/per_sample], and the two
  // host-rounded weights phi, psi = fl32(1 - phi). Only the <RS = true> instantiations read them.
  const float* ratio;
  float phi, psi;
  // per-sample classifier-free guidance (dpm_step_guided): fp32 scale per sample [n/per_sample], in place of
  // `guidance`. Only the <PG = true> instantiations read it; with it, `ratio` may be NULL (no rescale).
  const float* gscale;
  // FLOW and EDM (direct_param): the conversion v = conv_a*xe + conv_b*out of the packet kernels (flow8), formed on the
  // host from param, predict_x0 and the by-value alpha_e, sigma_e (build_params). Only flow8 reads them.
  float conv_a, conv_b;
  // adaptive projected guidance (dpm_step_apg): the per-sample words A_b = apg_a[b], B_b = apg_b[b] of dpm_apg_words,
  // the fp32 guidance direction R (NULL: R = x0_c - x0_u from e_uncond), and the marginals of the x0 -> eps conversion
  // (predict_x0 == 0). `gscale`, when set, marks the samples whose scale is 1 (bypass). Only the <APG = true>
  // instantiations read them.
  const float* apg_a;
  const float* apg_b;
  const float* apg_r;
  float apg_alpha, apg_sigma;
  // CFG-Zero* (dpm_step_cfgzero): the per-sample optimised scale s*_b of dpm_cfgzero_scale, fp32 [n/per_sample]. Only
  // the <PG = true> instantiations read it (kind kPgZeroStar); `gscale` may then be NULL (every sample's scale is
  // `guidance`).
  const float* zs;
  // TCFG (dpm_step_tcfg): the per-sample words (wu_b, wc_b) of dpm_tcfg_words, fp32 [n/per_sample][2]. Only the
  // <PG = true> instantiations read it (kind kPgTangential); `gscale` may then be NULL (every sample's scale is
  // `guidance`).
  const float* td;
};

// multi-condition classifier-free guidance (dpm_step_multi): eps = eps_u; eps = eps + s[k]*(eps_k - eps_u) for k < n_cond,
// each output converted by the parameterisation first. `k.eu` is the unconditional output; `k.ec` and `k.out2` are not
// read. rep[k] (optional) receives x_t again: block k + 1 of the [(n_cond + 1)B, ...] network input. KParams itself is
// left as it is, so the kernels that take it keep their code.
constexpr int kMaxCond = DPM_MAX_CONDITIONS;
struct MultiParams {
  KParams k;
  const void* ec[kMaxCond];
  void* rep[kMaxCond];
  float s[kMaxCond];
  int32_t n_cond;
};

// regional multi-condition guidance (dpm_step_multi_masked): MultiParams with one weight map per condition, the weight
// of s[k] at global element i being w[k][b*sstride[k] + (i - b*k.per_sample) % period[k]], b = i / k.per_sample
// (w[k] NULL: 1). MultiParams stays as it is, so k_step_multi keeps its code.
struct MaskedParams {
  MultiParams m;
  const float* w[kMaxCond];
  uint64_t period[kMaxCond];
  uint64_t sstride[kMaxCond];
};

// UniPC (dpm_step_unipc): the corrector of step i and the predictor of step i+1 around the conversion of KParams, whose
// own update fields (form, a, c*, w*) are not read. k.x is x~_i (also the evaluation state), k.m0 m_i when n_model == 0,
// k.m1 / k.m2 / m3 the buffers m_{i-1} / m_{i-2} / m_{i-3}; out_c (optional) receives the corrected x_i.
struct UniParams {
  KParams k;
  const void* m3;
  void* out_c;
  int32_t pc, pp;      // corrector order 0..3 (0 = off), predictor order 0..3 (0 = none)
  float cd[2], ct;     // corrector words
  float a, c0, cp[2];  // predictor words
};
// CFG++ (dpm_step_cfgpp): a LIN1 or multistep DIFF2 update of a CFG pair (KParams as dpm_step builds it; gscale NULL
// or the per-sample scales) that buffers the unguided x0 and adds g*(G - U); g = alpha_t of the step's end time.
struct CfgppParams {
  KParams k;
  float g;
};

// the buffers a UniPC launch reads: m_{i-1} for the corrector or a predictor of order >= 2, m_{i-2} for a corrector of
// order >= 2 or a predictor of order 3, m_{i-3} for a corrector of order 3
struct UniReads {
  bool m1, m2, m3;
};
__host__ __device__ __forceinline__ UniReads uni_reads(int pc, int pp) {
  return {pc >= 1 || pp >= 2, pc >= 2 || pp >= 3, pc >= 3};
}

// ---- storage types ------------------------------------------------------------------------
template <typename T> struct Raw;  // one packet as loaded (still packed)
template <> struct Raw<float> { uint32_t r[8]; };
template <> struct Raw<__nv_bfloat16> { uint32_t r[4]; };
template <> struct Raw<__half> { uint32_t r[4]; };

template <typename T> struct Traits;
template <> struct Traits<float> { static constexpr int kBytes = 4; static constexpr int kCode = DPM_F32; };
template <> struct Traits<__nv_bfloat16> { static constexpr int kBytes = 2; static constexpr int kCode = DPM_BF16; };
template <> struct Traits<__half> { static constexpr int kBytes = 2; static constexpr int kCode = DPM_F16; };

// Streaming global access: bypass L1 allocation (each byte is touched once per launch).
// Plain (coherent) ld.global so that `out` may alias `x` element-wise.
// sm_90 has no 256-bit global access: an fp32 packet is two 128-bit accesses (LDG.E.128) to the
// two halves of one 32-byte sector.
__device__ __forceinline__ void ldg_pk(Raw<float>& v, const float* p) {
  asm volatile("ld.global.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.L1::no_allocate.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(v.r[0]), "=r"(v.r[1]), "=r"(v.r[2]), "=r"(v.r[3]), "=r"(v.r[4]),
                 "=r"(v.r[5]), "=r"(v.r[6]), "=r"(v.r[7])
               : "l"(p));
}
template <typename T16>
__device__ __forceinline__ void ldg_pk(Raw<T16>& v, const T16* p) {
  asm volatile("ld.global.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.r[0]), "=r"(v.r[1]), "=r"(v.r[2]), "=r"(v.r[3])
               : "l"(p));
}
__device__ __forceinline__ void stg_pk(float* p, const Raw<float>& v) {
  asm volatile("st.global.L1::no_allocate.v4.b32 [%0], {%1,%2,%3,%4};\n\t"
               "st.global.L1::no_allocate.v4.b32 [%0+16], {%5,%6,%7,%8};" ::"l"(p),
               "r"(v.r[0]), "r"(v.r[1]), "r"(v.r[2]), "r"(v.r[3]), "r"(v.r[4]), "r"(v.r[5]),
               "r"(v.r[6]), "r"(v.r[7])
               : "memory");
}
template <typename T16>
__device__ __forceinline__ void stg_pk(T16* p, const Raw<T16>& v) {
  asm volatile("st.global.L1::no_allocate.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.r[0]),
               "r"(v.r[1]), "r"(v.r[2]), "r"(v.r[3])
               : "memory");
}

// unpack / pack -----------------------------------------------------------------------------
__device__ __forceinline__ void unpack(const Raw<float>& v, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = __uint_as_float(v.r[i]);
}
__device__ __forceinline__ void unpack(const Raw<__nv_bfloat16>& v, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    f[2 * i] = __uint_as_float(v.r[i] << 16);
    f[2 * i + 1] = __uint_as_float(v.r[i] & 0xffff0000u);
  }
}
__device__ __forceinline__ void unpack(const Raw<__half>& v, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = *reinterpret_cast<const __half2*>(&v.r[i]);
    float2 t = __half22float2(h);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ void pack(Raw<float>& v, const float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) v.r[i] = __float_as_uint(f[i]);
}
__device__ __forceinline__ void pack(Raw<__nv_bfloat16>& v, const float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    v.r[i] = *reinterpret_cast<uint32_t*>(&h);
  }
}
__device__ __forceinline__ void pack(Raw<__half>& v, const float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    v.r[i] = *reinterpret_cast<uint32_t*>(&h);
  }
}

// value as it will read back from storage (so fused and unfused paths agree bit for bit)
template <typename T> __device__ __forceinline__ float round_storage(float v);
template <> __device__ __forceinline__ float round_storage<float>(float v) { return v; }
template <> __device__ __forceinline__ float round_storage<__nv_bfloat16>(float v) {
  return __bfloat162float(__float2bfloat16_rn(v));
}
template <> __device__ __forceinline__ float round_storage<__half>(float v) {
  return __half2float(__float2half_rn(v));
}

// dtype-generic scalar access (generic kernel, quantile fallback)
__device__ __forceinline__ float load_any(const void* p, int dt, size_t i) {
  switch (dt) {
    case DPM_BF16: return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
    case DPM_F16: return __half2float(static_cast<const __half*>(p)[i]);
    default: return static_cast<const float*>(p)[i];
  }
}
__device__ __forceinline__ float store_any(void* p, int dt, size_t i, float v) {
  switch (dt) {
    case DPM_BF16: {
      __nv_bfloat16 h = __float2bfloat16_rn(v);
      static_cast<__nv_bfloat16*>(p)[i] = h;
      return __bfloat162float(h);
    }
    case DPM_F16: {
      __half h = __float2half_rn(v);
      static_cast<__half*>(p)[i] = h;
      return __half2float(h);
    }
    default: static_cast<float*>(p)[i] = v; return v;
  }
}
__device__ __forceinline__ float round_any(int dt, float v) {
  switch (dt) {
    case DPM_BF16: return round_storage<__nv_bfloat16>(v);
    case DPM_F16: return round_storage<__half>(v);
    default: return v;
  }
}

// ---- exact division by a launch constant -------------------------------------------------------
// x / d for a divisor that is uniform over the launch, without the per-element IEEE division
// subroutine (MUFU.RCP + 4 FFMA + FCHK + slow-path call). With r = RN(1/d) prepared once:
//   q0 = RN(x*r); e = x - q0*d (one FMA); q1 = RN(q0 + e*r); repeat once.
// q0 can be up to ~1.4 ulp from x/d (half an ulp of r's error scaled to the quotient plus the product's
// rounding), so its residual need not be exact; q1 is faithful (within an ulp), the residual of a
// faithful quotient IS exact in one FMA, and Markstein's division theorem then makes the second
// refinement the correctly rounded quotient -- provided d's significand is not all ones (checked on
// the host, recip_div_ok) and nothing under/overflows in the residual, guarded below by routing
// tiny/huge/non-finite/zero x to the IEEE division. (One refinement alone matched IEEE on 4e8 random
// pairs but is not provable: its error bound, 1.7e-7 ulp, exceeds the closest a quotient can come to
// a rounding midpoint, 1.5e-8 ulp.) tests/test_gpu_kernels.py::test_constant_division_is_ieee compares
// it bit for bit with true division over ~10^9 (x, d) pairs; tests/test_math_properties.py repeats the
// argument in exact rational arithmetic. Explicit fmaf() stays fused under -fmad=false.
static __device__ __noinline__ float div_ieee_cold(float x, float d) { return x / d; }

__device__ __forceinline__ float div_const(float x, float d, float r) {
  float q = x * r;
  float e = fmaf(-q, d, x);
  q = fmaf(e, r, q);
  e = fmaf(-q, d, x);
  q = fmaf(e, r, q);
  const float ax = fabsf(x);
  if (!(ax > 1e-25f && ax < 1e30f)) q = div_ieee_cold(x, d);  // zero, tiny, huge, inf, nan: IEEE path
  return q;
}
// packet form: the range guard is one min and one max over the 8 magnitudes (a NaN that the min/max
// skip still comes out of the refinement as NaN) and one never-inlined IEEE call site per element,
// off the hot path
__device__ __forceinline__ void div_const8(float (&x)[8], float d, float r) {
  float q[8];
  float mn = fabsf(x[0]), mx = mn;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float t = x[i] * r;
    float e = fmaf(-t, d, x[i]);
    t = fmaf(e, r, t);
    e = fmaf(-t, d, x[i]);
    q[i] = fmaf(e, r, t);
    if (i > 0) {
      mn = fminf(mn, fabsf(x[i]));
      mx = fmaxf(mx, fabsf(x[i]));
    }
  }
  if (!(mn > 1e-25f && mx < 1e30f)) {
#pragma unroll
    for (int i = 0; i < 8; ++i) q[i] = div_ieee_cold(x[i], d);   // fully unrolled: a dynamic index would put q[] in local memory
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) x[i] = q[i];
}
__host__ __device__ __forceinline__ bool recip_div_ok(float d) {
  // |d| in [2^-20, 2^21), biased exponent 107..147 (so that with 1e-25 < |x| < 1e30 neither the quotient nor
  // the residual of div_const can overflow or reach the denormal range), significand not all ones
#ifdef __CUDA_ARCH__
  const uint32_t b = __float_as_uint(d);
#else
  uint32_t b;
  memcpy(&b, &d, 4);
#endif
  const uint32_t ex = (b >> 23) & 0xffu;
  return ex >= 107u && ex <= 147u && (b & 0x7fffffu) != 0x7fffffu;
}

// ---- per-element arithmetic -----------------------------------------------------------------
// torch.clamp(x0, -s, s) (:424) for s >= 0, NaN-propagating like ATen's clamp: fminf/fmaxf would turn a NaN x0
// into -s; with comparisons a NaN x0 (every comparison false) passes through, and a NaN s reaches the result
// through the division that follows.
__device__ __forceinline__ float clamp_sym(float x0, float s) {
  return x0 > s ? s : (x0 < -s ? -s : x0);
}
// torch.maximum / Tensor.max(): NaN wins
__device__ __forceinline__ float max_nan(float a, float b) {
  return (a != a) ? a : ((b != b) ? b : fmaxf(a, b));
}
// torch.min(a, b) / torch.minimum: NaN wins; otherwise std::min's `b < a ? b : a`
__device__ __forceinline__ float min_nan(float a, float b) {
  return (a != a) ? a : ((b != b) ? b : (b < a ? b : a));
}
// DPM_PARAM_FLOW: the velocity of a flow-matching model, converted straight into the solver's space (no division)
__device__ __forceinline__ float flow_value(bool x0, float out, float xe, float alpha, float sigma) {
  return x0 ? xe - sigma * out : xe + alpha * out;
}
// FLOW and EDM convert straight into the solver's space: x0 when p.predict_x0, else eps, with no eps -> x0 division
__host__ __device__ __forceinline__ bool direct_param(int param) {
  return param == DPM_PARAM_FLOW || param == DPM_PARAM_EDM;
}
// model_wrapper.noise_pred_fn :288-298. FLOW and EDM return x0 when p.predict_x0 and eps otherwise (finish_x0 then skips
// :439); EDM's alpha_e / sigma_e are the host words of that space.
__device__ __forceinline__ float convert_param(const KParams& p, float out, float xe) {
  const float alpha = p.alpha_e, sigma = p.sigma_e;
  switch (p.param) {
    case DPM_PARAM_X_START: return (xe - alpha * out) / sigma;   // :292
    case DPM_PARAM_V: return alpha * out + sigma * xe;           // :295
    case DPM_PARAM_SCORE: return (-sigma) * out;                 // :298
    case DPM_PARAM_FLOW: return flow_value(p.predict_x0 != 0, out, xe, alpha, sigma);
    case DPM_PARAM_EDM: return alpha * xe + sigma * out;
    default: return out;                                         // :289
  }
}
// converted and combined prediction -> buffered model value: eps, or x0 (:439, the thresholding clamp :424)
__device__ __forceinline__ float finish_x0(const KParams& p, float eps, float xe, float thr, bool clamp) {
  if (!p.predict_x0) return eps;
  float x0 = direct_param(p.param) ? eps : (xe - p.sigma_e * eps) / p.alpha_e;  // data_prediction_fn :439
  if (clamp) x0 = clamp_sym(x0, thr) / thr;  // dynamic_thresholding_fn :424
  return x0;
}

// raw network output(s) -> buffered model value (eps, or x0 for dpmsolver++)
// RND: reference-rounding mode. A network that returns 16-bit noise makes the reference evaluate the
// CFG combine in that type (python-float scale, :329-330): three ops, each rounded to 16 bits.
// guidance rescale (Lin et al. 2023; diffusers' rescale_noise_cfg), in the network's output space:
// g' = phi*(g*r) + psi*g, r = std(out_c)/std(g) of the sample, each op rounded
__device__ __forceinline__ float rescale_value(const KParams& p, float g, float r) {
  return p.phi * (g * r) + p.psi * g;
}

// per-sample guidance with the sample's scale gs, in one of three kinds that are uniform over a sample (the caller
// picks the kind once per packet, or per element with kPgAny):
//   kPgBypass  gs == 1: the reference's bypass (:323), the converted conditional output alone (no combine, no rescale)
//   kPgRescale p.ratio set: the rescaled combine of the RS path
//   kPgCombine otherwise: the combine of the plain path
//   kPgZeroStar p.zs set: CFG-Zero* (Fan et al. 2025) in the network's output space with r = s*_b of the sample:
//              us = eu*s*, g = us + gs*(ec - us), each op rounded, then the parameterisation converts g
//   kPgTangential p.td set: TCFG (tangential damping, CVPR 2025) in the network's output space with r, r2 = the
//              words wu_b, wc_b of the sample: us = eu*wu + ec*wc, g = us + gs*(ec - us), each op rounded, then the
//              parameterisation converts g
// Precedence: the bypass, then zs, td, ratio, the plain combine.
enum { kPgAny = 1, kPgBypass = 2, kPgRescale = 3, kPgCombine = 4, kPgZeroStar = 5, kPgTangential = 6 };
__host__ __device__ __forceinline__ int pg_kind(const KParams& p, float gs) {
  if (gs == 1.f) return kPgBypass;
  if (p.zs != nullptr) return kPgZeroStar;
  if (p.td != nullptr) return kPgTangential;
  return p.ratio != nullptr ? kPgRescale : kPgCombine;
}
template <int K>
__device__ __forceinline__ float guided_value(const KParams& p, float xe, float ec, float eu, float r, float gs,
                                              float r2) {
  if constexpr (K == kPgAny) {
    const int k = pg_kind(p, gs);
    if (k == kPgBypass) return guided_value<kPgBypass>(p, xe, ec, eu, r, gs, r2);
    if (k == kPgRescale) return guided_value<kPgRescale>(p, xe, ec, eu, r, gs, r2);
    if (k == kPgZeroStar) return guided_value<kPgZeroStar>(p, xe, ec, eu, r, gs, r2);
    if (k == kPgTangential) return guided_value<kPgTangential>(p, xe, ec, eu, r, gs, r2);
    return guided_value<kPgCombine>(p, xe, ec, eu, r, gs, r2);
  } else if constexpr (K == kPgBypass) {
    return convert_param(p, ec, xe);
  } else if constexpr (K == kPgRescale) {
    return convert_param(p, rescale_value(p, eu + gs * (ec - eu), r), xe);
  } else if constexpr (K == kPgZeroStar) {
    const float us = eu * r;
    return convert_param(p, us + gs * (ec - us), xe);
  } else if constexpr (K == kPgTangential) {
    const float us = eu * r + ec * r2;
    return convert_param(p, us + gs * (ec - us), xe);
  } else {
    const float epc = convert_param(p, ec, xe);
    const float epu = convert_param(p, eu, xe);
    return epu + gs * (epc - epu);  // :330
  }
}

// RS: guidance rescale (NE == 2). The combine then runs on the raw outputs, the rescale follows, and the
// parameterisation converts the rescaled prediction -- the order of a rescaling network wrapped by :288-298.
// PG: per-sample guidance (NE == 2, guided_value<PG>) with the sample's scale gs; 0 = off, else the kind. r2: the
// second word of the sample (kPgTangential).
template <int NE, bool RND = false, bool RS = false, int PG = 0>
__device__ __forceinline__ float model_value(const KParams& p, float xe, float ec, float eu,
                                             float thr, bool clamp, float r = 1.f, float gs = 1.f, float r2 = 0.f) {
  float eps;
  if constexpr (PG != 0) {
    eps = guided_value<PG>(p, xe, ec, eu, r, gs, r2);
  } else if (RS) {
    eps = convert_param(p, rescale_value(p, eu + p.guidance * (ec - eu), r), xe);
  } else {
    eps = convert_param(p, ec, xe);
  }
  if (NE == 2 && !RS && !PG) {
    float epu = convert_param(p, eu, xe);
    if (RND && p.param == DPM_PARAM_NOISE) {
      const int dt = p.raw_round & 3;
      const float d = round_any(dt, eps - epu);
      eps = round_any(dt, epu + round_any(dt, p.guidance * d));
    } else {
      eps = epu + p.guidance * (eps - epu);  // model_wrapper.model_fn :330
    }
  }
  return finish_x0(p, eps, xe, thr, clamp);
}

// ---- adaptive projected guidance (Sadat et al. 2025) ------------------------------------------------------------
// one network output -> the denoised prediction by the step's parameterisation, each op rounded: FLOW x0 = xe -
// sigma_e*out, EDM alpha_e*xe + sigma_e*out with the x0 words, every other one converted to eps (:288-298) and then to
// x0 (:439). alpha_e, sigma_e are those of a predict_x0 step, whatever the launch buffers.
__device__ __forceinline__ float apg_x0(const KParams& p, float out, float xe) {
  if (p.param == DPM_PARAM_FLOW) return xe - p.sigma_e * out;
  const float v = convert_param(p, out, xe);
  return p.param == DPM_PARAM_EDM ? v : (xe - p.sigma_e * v) / p.alpha_e;
}
// the guided denoised prediction A*c + B*R (c for a bypassed sample), then the buffered value: x0 with the clamp
// (:424), or eps by the x_start conversion with the marginals apg_alpha, apg_sigma (:292). `ru` is R when has_r, else
// the unconditional output.
__device__ __forceinline__ float apg_value(const KParams& p, float xe, float ec, float ru, bool has_r, float A, float B,
                                           bool bypass, float thr, bool clamp) {
  const float c = apg_x0(p, ec, xe);
  float g = c;
  if (!bypass) {
    const float R = has_r ? ru : c - apg_x0(p, ru, xe);
    g = A * c + B * R;
  }
  if (p.predict_x0) return clamp ? clamp_sym(g, thr) / thr : g;
  return (xe - p.apg_alpha * g) / p.apg_sigma;
}

// round a packet to its storage type once: returns the packed words and rewrites f[] with the
// values as they will read back (so fused and unfused paths agree bit for bit)
__device__ __forceinline__ void round_pack(Raw<float>& r, float (&f)[8]) { pack(r, f); }
template <typename T16>
__device__ __forceinline__ void round_pack(Raw<T16>& r, float (&f)[8]) {
  pack(r, f);
  unpack(r, f);
}

// the update. T0 = newest model value, m1/m2 = older buffers.
// RND: reference-rounding mode, bit 2: the buffered values are raw 16-bit network outputs, so the
// reference forms their differences (:823, :880-881, :636, :735, :741-742) in that type.
template <int FORM, bool RND = false>
__device__ __forceinline__ float update_value(const KParams& p, float x, float T0, float m1,
                                              float m2) {
  const int ddt = (RND && (p.raw_round & 4)) ? (p.raw_round & 3) : DPM_F32;
  auto diff = [&](float u, float v) { return RND ? round_any(ddt, u - v) : u - v; };
  if (FORM == DPM_FORM_LIN1) {
    return p.a * x + p.c0 * T0;  // :573-576 / :585-588
  } else if (FORM == DPM_FORM_LIN2) {
    return (p.a * x + p.c0 * T0) + p.c1 * m1;
  } else if (FORM == DPM_FORM_LIN3) {
    return ((p.a * x + p.c0 * T0) + p.c1 * m1) + p.c2 * m2;
  } else if (FORM == DPM_FORM_DIFF2) {
    float D = p.w0 * diff(T0, m1);           // :823 (w0 = 1/r0) or :639 (w0 = 1)
    float lead = p.c0_on_old ? m1 : T0;      // singlestep: coefficient sits on model_s
    return (p.a * x + p.c0 * lead) + p.c1 * D;  // :827-851, :636-669, :728-739
  } else if (FORM == DPM_FORM_MS3) {
    float D10 = p.w0 * diff(T0, m1);   // :880
    float D11 = p.w1 * diff(m1, m2);   // :881
    float dd = D10 - D11;
    float D1 = D10 + p.w2 * dd;     // :882
    float D2 = p.w3 * dd;           // :883
    return ((p.a * x + p.c0 * T0) + p.c1 * D1) + p.c2 * D2;  // :888-893 / :898-903
  } else if (FORM == DPM_FORM_SS3T) {
    // m2 = model_s, m1 = model_s1, T0 = model_s2
    if (RND && (p.raw_round & 4)) {
      // r1, r2 are python floats or 0-dim tensors (:741-744, :780-783): they do not promote, so with raw
      // 16-bit buffers the reference evaluates D1 and D2 entirely in that type, one rounding per op
      auto R = [&](float v) { return round_any(ddt, v); };
      const float D10 = R(p.w0 * R(m1 - m2)), D11 = R(p.w1 * R(T0 - m2));
      const float D1 = R(R(R(p.w2 * D10) - R(p.w3 * D11)) / p.w4);
      const float D2 = R(R(2.f * R(D11 - D10)) / p.w4);
      return ((p.a * x + p.c0 * m2) + p.c1 * D1) + p.c2 * D2;
    }
    float D10 = p.w0 * (m1 - m2);                 // :741
    float D11 = p.w1 * (T0 - m2);                 // :742
    float n1 = p.w2 * D10 - p.w3 * D11, n2 = 2.f * (D11 - D10);
    float D1 = p.fast_div ? div_const(n1, p.w4, p.r_w4) : n1 / p.w4;  // :743
    float D2 = p.fast_div ? div_const(n2, p.w4, p.r_w4) : n2 / p.w4;  // :744
    return ((p.a * x + p.c0 * m2) + p.c1 * D1) + p.c2 * D2;  // :745-750 / :784-789
  }
  return 0.f;
}

// ---- the fast path: noise-, flow- and EDM-parameterised networks, exact constant division ------
// Launch-uniform switches are taken once per PACKET (uniform branches), every loop below is
// straight-line code over 8 elements. Callers guarantee: p.param == NOISE, FLOW or EDM; p.fast_div when a division
// is needed (a FLOW or EDM conversion has none); a clamp threshold `s` that is uniform over the packet.
// FLOW and EDM convert each output first (flow8, in the solver's space) and combine the converted values; a rescaled
// combine runs on the raw outputs and is converted afterwards. ec and eu are overwritten.
// Both are one affine map v = conv_a*xe + conv_b*v with launch-uniform words (KParams::conv_a, conv_b): EDM's
// (alpha_e, sigma_e), and for FLOW conv_a = 1 with conv_b = -sigma_e (x0) or alpha_e (eps). 1*xe is xe and
// xe + (-s)*v is xe - s*v exactly, zeros and NaNs included, so a FLOW value is bit for bit flow_value's.
__device__ __forceinline__ void flow8(const KParams& p, const float (&xe)[8], float (&v)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = p.conv_a * xe[i] + p.conv_b * v[i];
}
// combined prediction T -> buffered model value: eps -> x0 (:439; a FLOW or EDM value is x0 already) and the clamp (:424)
__device__ __forceinline__ void fast_finish8(const KParams& p, const float (&xe)[8], bool clamp, float s, float (&T)[8]) {
  if (!p.predict_x0) return;
  if (!direct_param(p.param)) {
#pragma unroll
    for (int i = 0; i < 8; ++i) T[i] = xe[i] - p.sigma_e * T[i];
    div_const8(T, p.alpha_e, p.r_alpha);  // :439
  }
  if (clamp) {
#pragma unroll
    for (int i = 0; i < 8; ++i) T[i] = clamp_sym(T[i], s);
    if (recip_div_ok(s)) {
      div_const8(T, s, __frcp_rn(s));  // :424
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) T[i] = div_ieee_cold(T[i], s);
    }
  }
}
// RS: guidance rescale with the sample's ratio r (uniform over the packet, like s).
// PG: per-sample guidance with the sample's scale gs (uniform over the packet): gs == 1 selects ec (the bypass),
// else the combine, rescaled when p.ratio is set -- both branches uniform per packet.
template <int NE, bool RS = false, bool PG = false>
__device__ __forceinline__ void fast_model8(const KParams& p, const float (&xe)[8], float (&ec)[8],
                                            float (&eu)[8], bool clamp, float s, float (&T)[8],
                                            float r = 1.f, float gs = 1.f) {
  const bool flow = direct_param(p.param);
  const bool raw_combine = RS || (PG && p.ratio != nullptr);   // rescaled: combine the raw outputs, convert after
  if (flow && !raw_combine) {
    flow8(p, xe, ec);
    if (NE == 2) flow8(p, xe, eu);
  }
  if constexpr (PG) {
    if (gs == 1.f) {
#pragma unroll
      for (int i = 0; i < 8; ++i) T[i] = ec[i];   // :323 (NOISE: the conversion is the identity; FLOW, EDM: done above or below)
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) T[i] = eu[i] + gs * (ec[i] - eu[i]);  // :330
      if (p.ratio != nullptr) {
#pragma unroll
        for (int i = 0; i < 8; ++i) T[i] = rescale_value(p, T[i], r);
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) T[i] = (NE == 2) ? eu[i] + p.guidance * (ec[i] - eu[i]) : ec[i];  // :330
  }
  if (RS) {
#pragma unroll
    for (int i = 0; i < 8; ++i) T[i] = rescale_value(p, T[i], r);
  }
  if (flow && raw_combine) flow8(p, xe, T);
  fast_finish8(p, xe, clamp, s, T);
}

template <int FORM>
__device__ __forceinline__ void fast_update8(const KParams& p, const float (&x)[8], const float (&T)[8],
                                             const float (&m1)[8], const float (&m2)[8], float (&o)[8]) {
  if (FORM == DPM_FORM_DIFF2) {
    // the coefficient sits on model_s for the singlestep difference steps: one uniform branch per packet
    if (p.c0_on_old) {
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = (p.a * x[i] + p.c0 * m1[i]) + p.c1 * (p.w0 * (T[i] - m1[i]));  // :636-669, :728-739
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = (p.a * x[i] + p.c0 * T[i]) + p.c1 * (p.w0 * (T[i] - m1[i]));   // :823-851
    }
  } else if (FORM == DPM_FORM_SS3T) {
    float n1[8], n2[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float D10 = p.w0 * (m1[i] - m2[i]);  // :741
      const float D11 = p.w1 * (T[i] - m2[i]);   // :742
      n1[i] = p.w2 * D10 - p.w3 * D11;
      n2[i] = 2.f * (D11 - D10);
    }
    div_const8(n1, p.w4, p.r_w4);  // :743
    div_const8(n2, p.w4, p.r_w4);  // :744
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = ((p.a * x[i] + p.c0 * m2[i]) + p.c1 * n1[i]) + p.c2 * n2[i];  // :745-750 / :784-789
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = update_value<FORM>(p, x[i], T[i], m1[i], m2[i]);
  }
}

// launch-time test: can this request run on the <FAST = true> instantiations?
__host__ __forceinline__ bool fast_path_ok(const KParams& p) {
  if (p.form == DPM_FORM_SS3T && !p.fast_div) return false;
  if (p.n_model == 0) return true;
  if (p.param != DPM_PARAM_NOISE && !direct_param(p.param)) return false;
  if (p.param == DPM_PARAM_NOISE && p.predict_x0 && !p.fast_div) return false;   // FLOW, EDM: no division by alpha_e
  if ((p.thr != nullptr || p.ratio != nullptr || p.gscale != nullptr) && p.pk_per_sample == 0) return false;
  return true;
}

// the state and buffer streams a form reads: the kernels (at compile time), the generic kernel, the TMA stage
// layout and the host-side argument and alignment checks all take them from here
struct FormReads {
  bool x, m1, m2;
};
__host__ __device__ constexpr FormReads form_reads(int form) {
  return {form != DPM_FORM_NONE,
          form == DPM_FORM_LIN2 || form == DPM_FORM_LIN3 || form == DPM_FORM_DIFF2 || form == DPM_FORM_MS3 ||
              form == DPM_FORM_SS3T,
          form == DPM_FORM_LIN3 || form == DPM_FORM_MS3 || form == DPM_FORM_SS3T};
}

}  // namespace dpm
