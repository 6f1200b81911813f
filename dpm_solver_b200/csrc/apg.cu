// apg.cu -- the per-sample words of adaptive projected guidance (dpm_apg_words; Sadat, Hilliges and Weber,
// "Eliminating Oversaturation and Artifacts of High Guidance Scales in Diffusion Models", ICLR 2025):
//   c = x0(out_c), u = x0(out_u), D = c - u                       (the step's conversion, each op rounded)
//   R = D, or R = D + beta*R_prev                                  (momentum; written to r_out when set)
//   k = min(1, r/||R||) (r > 0), p = <R, c>/max(||c||, 1e-12)^2
//   A = 1 - (w - 1)*(1 - eta)*k*p,  B = (w - 1)*k                  (fp64, each rounded to fp32 once)
// so that the step's guided prediction c + (w - 1)*(k*R - (1 - eta)*k*p*c) is A*c + B*R.
// Same chunking as the rescale ratio (adaptive.cu): CTA (b, c) reduces chunk c of sample b to three fp64 partials, the
// final kernel merges a sample's chunks in chunk order. Every thread owns the same elements on the vector and the
// element-wise path and every sum runs in a fixed order, so the words of sample b depend on its values only.
// Algorithmic bytes per element: x, out_c, out_u read, plus 4 + 4 of R_prev / R with momentum.
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kAThreads = 256;
constexpr int kAChunk = 8192;   // elements per CTA

struct AParams {
  KParams k;             // xe, ec, eu, param, alpha_e, sigma_e (x0 words), guidance, dtypes, dev_coef
  const float* gscale;   // per-sample scales [n_samples], or NULL: k.guidance
  const float* r_prev;   // NULL: R = D
  float* r_out;          // NULL: R is not written
  double* partial;       // [n_samples * chunks][3]: ||R||^2, <R, c>, ||c||^2
  float* words;          // [2][n_samples]
  uint64_t per_sample;
  uint64_t n_samples;
  uint32_t chunks;       // per sample
  float eta, norm_threshold, momentum;
};

// deterministic CTA sum of one double per thread (butterfly within the warps, then the warps in order)
__device__ __forceinline__ double apg_cta_sum(double v, double* warp_part) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();   // warp_part may still be read from the previous call
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < kAThreads / 32; ++w) s += warp_part[w];
  return s;
}

// VEC: per_sample % 8 == 0 and every operand aligned; TE, TS the packet pair. Otherwise element-wise (load_any).
template <typename TE, typename TS, bool VEC>
__global__ void __launch_bounds__(kAThreads) k_apg_partial(const __grid_constant__ AParams p) {
  __shared__ double warp_part[kAThreads / 32];
  KParams k = p.k;
  if (k.dev_coef != nullptr) { k.alpha_e = k.dev_coef[9]; k.sigma_e = k.dev_coef[10]; }
  const uint64_t sample = blockIdx.x / p.chunks;
  const uint32_t chunk = blockIdx.x % p.chunks;
  const uint64_t c_begin = (uint64_t)chunk * kAChunk;
  const uint64_t c_end = c_begin + kAChunk < p.per_sample ? c_begin + kAChunk : p.per_sample;
  const uint32_t cnt = (uint32_t)(c_end - c_begin);
  const size_t e0 = sample * p.per_sample + c_begin;
  const int tid = threadIdx.x;
  constexpr int U = kAChunk / kPacket / kAThreads;   // 4
  double srr = 0.0, src = 0.0, scc = 0.0;
  auto term = [&](float xe, float oc, float ou, float rp, float& R) {
    const float c = apg_x0(k, oc, xe);
    const float D = c - apg_x0(k, ou, xe);
    R = p.r_prev != nullptr ? D + p.momentum * rp : D;
    srr += (double)R * (double)R;
    src += (double)R * (double)c;
    scc += (double)c * (double)c;
  };
  // element (u, i) of this thread is chunk element (u*kAThreads + tid)*8 + i on both paths
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const uint32_t pk = u * kAThreads + tid;
    if (VEC) {
      if (pk * kPacket < cnt) {
        const size_t e = e0 + (size_t)pk * kPacket;
        Raw<TS> rx;
        Raw<TE> rc, ru;
        Raw<float> rp;
        ldg_pk(rx, static_cast<const TS*>(k.xe) + e);
        ldg_pk(rc, static_cast<const TE*>(k.ec) + e);
        ldg_pk(ru, static_cast<const TE*>(k.eu) + e);
        if (p.r_prev != nullptr) ldg_pk(rp, p.r_prev + e);
        float fx[8], fc[8], fu[8], fp[8], fr[8];
        unpack(rx, fx);
        unpack(rc, fc);
        unpack(ru, fu);
        if (p.r_prev != nullptr) unpack(rp, fp);
#pragma unroll
        for (int i = 0; i < 8; ++i) term(fx[i], fc[i], fu[i], p.r_prev != nullptr ? fp[i] : 0.f, fr[i]);
        if (p.r_out != nullptr) {
          Raw<float> ro;
          pack(ro, fr);
          stg_pk(p.r_out + e, ro);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t j = pk * kPacket + i;
        if (j < cnt) {
          const size_t e = e0 + j;
          float R;
          term(load_any(k.xe, k.state_dtype, e), load_any(k.ec, k.model_dtype, e), load_any(k.eu, k.model_dtype, e),
               p.r_prev != nullptr ? p.r_prev[e] : 0.f, R);
          if (p.r_out != nullptr) p.r_out[e] = R;
        }
      }
    }
  }
  srr = apg_cta_sum(srr, warp_part);
  src = apg_cta_sum(src, warp_part);
  scc = apg_cta_sum(scc, warp_part);
  if (tid == 0) {
    double* o = p.partial + (size_t)blockIdx.x * 3;
    o[0] = srr; o[1] = src; o[2] = scc;
  }
}

__global__ void __launch_bounds__(kAThreads) k_apg_final(const __grid_constant__ AParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kAThreads + threadIdx.x;
  if (b >= p.n_samples) return;
  const double* part = p.partial + b * p.chunks * 3;
  double srr = 0.0, src = 0.0, scc = 0.0;
  for (uint32_t c = 0; c < p.chunks; ++c) {
    srr += part[c * 3];
    src += part[c * 3 + 1];
    scc += part[c * 3 + 2];
  }
  double kk = 1.0;
  if (p.norm_threshold > 0.f) {
    const double q = (double)p.norm_threshold / sqrt(srr);
    kk = q < 1.0 ? q : 1.0;
  }
  const double sc = sqrt(scc);
  const double nc = sc < 1e-12 ? 1e-12 : sc;                 // F.normalize's epsilon (a NaN norm stays NaN)
  const double proj = src / (nc * nc);
  const double w = (double)(p.gscale != nullptr ? p.gscale[b] : p.k.guidance);
  const double A = 1.0 - (w - 1.0) * (1.0 - (double)p.eta) * kk * proj;
  const double B = (w - 1.0) * kk;
  p.words[b] = (float)A;
  p.words[p.n_samples + b] = (float)B;
}

size_t apg_workspace_bytes(uint64_t n_samples, uint64_t per_sample) {
  if (per_sample == 0 || n_samples == 0) return 0;
  const uint64_t chunks = (per_sample + kAChunk - 1) / kAChunk;
  return (size_t)(n_samples * chunks) * 3 * sizeof(double);
}

int launch_apg_words(float* words, const KParams& kp, const float* gscale, float eta, float norm_threshold,
                     float momentum, const float* r_prev, float* r_out, void* ws, size_t ws_bytes, cudaStream_t stream) {
  AParams p;
  memset(&p, 0, sizeof(p));
  p.k = kp;
  p.gscale = gscale; p.r_prev = r_prev; p.r_out = r_out; p.words = words;
  p.per_sample = kp.per_sample; p.n_samples = kp.n / kp.per_sample;
  p.chunks = (uint32_t)((p.per_sample + kAChunk - 1) / kAChunk);
  p.eta = eta; p.norm_threshold = norm_threshold; p.momentum = momentum;
  p.partial = static_cast<double*>(ws);
  if (ws == nullptr || ws_bytes < apg_workspace_bytes(p.n_samples, p.per_sample) ||
      (reinterpret_cast<uintptr_t>(ws) & 7)) {
    set_error("apg words: workspace too small or not 8-byte aligned");
    return DPM_ERR_ARG;
  }
  if (p.n_samples * p.chunks > 0x7fffffffull) { set_error("apg words: too many chunks"); return DPM_ERR_UNSUPPORTED; }
  auto al = [](const void* q, int dt) { return (reinterpret_cast<uintptr_t>(q) & (dt == DPM_F32 ? 31 : 15)) == 0; };
  const bool vec = p.per_sample % kPacket == 0 && al(kp.xe, kp.state_dtype) && al(kp.ec, kp.model_dtype) &&
                   al(kp.eu, kp.model_dtype) && (r_prev == nullptr || al(r_prev, DPM_F32)) &&
                   (r_out == nullptr || al(r_out, DPM_F32));
  typedef void (*AKernel)(const AParams);
  AKernel k = nullptr;
  if (vec) {
    k = with_packet_pair(kp.model_dtype, kp.state_dtype, [&](auto pair) -> AKernel {
      using Pair = decltype(pair);
      return k_apg_partial<typename Pair::TE, typename Pair::TS, true>;
    });
  }
  if (k == nullptr) k = k_apg_partial<float, float, false>;   // any dtype pair, alignment or sample size
  k<<<(unsigned)(p.n_samples * p.chunks), kAThreads, 0, stream>>>(p);
  k_apg_final<<<(unsigned)((p.n_samples + kAThreads - 1) / kAThreads), kAThreads, 0, stream>>>(p);
  count_launch();
  count_launch();
  return DPM_OK;
}

// ---- CFG-Zero* (dpm_cfgzero_scale; Fan, Zheng, Yeh and Liu, arXiv:2503.18886) -------------------------------------
// s*_b = fl32(<c_b, u_b> / (||u_b||^2 + 1e-8)) over the two raw network halves of sample b, fp64 sums of the widened
// outputs. The chunking, thread ownership and summation order of k_apg_partial / k_apg_final, with two sums of raw
// values in place of three of converted ones: no x, no marginals, no dev_coef. Algorithmic bytes: 2*s_model per element.
// ---- TCFG (dpm_tcfg_words; "TCFG: Tangential Damping Classifier-free Guidance", CVPR 2025) -------------------------
// The same pass with three sums, A = ||u||^2, B = <u, c>, C = ||c||^2, and k_tcfg_final in place of k_cfgzero_final:
// the words (wu, wc) of u' = wu*u + wc*c, the projection of u on the first right singular vector of [u; c].
struct ZParams {
  const void* ec;
  const void* eu;
  double* partial;       // [n_samples * chunks][NS]: <c, u>, ||u||^2 (CFG-Zero*) or ||u||^2, <u, c>, ||c||^2 (TCFG)
  float* s_out;          // [n_samples] s* (CFG-Zero*) or [n_samples][2] (wu, wc) (TCFG)
  uint64_t per_sample;
  uint64_t n_samples;
  uint32_t chunks;
  int32_t model_dtype;
};

// VEC: per_sample % 8 == 0 and both halves aligned, TE their type. Otherwise element-wise (load_any). NS: the number of
// sums, 2 (CFG-Zero*) or 3 (TCFG).
template <typename TE, bool VEC, int NS>
__global__ void __launch_bounds__(kAThreads) k_cfgzero_partial(const __grid_constant__ ZParams p) {
  static_assert(NS == 2 || NS == 3, "two or three sums");
  __shared__ double warp_part[kAThreads / 32];
  const uint64_t sample = blockIdx.x / p.chunks;
  const uint32_t chunk = blockIdx.x % p.chunks;
  const uint64_t c_begin = (uint64_t)chunk * kAChunk;
  const uint64_t c_end = c_begin + kAChunk < p.per_sample ? c_begin + kAChunk : p.per_sample;
  const uint32_t cnt = (uint32_t)(c_end - c_begin);
  const size_t e0 = sample * p.per_sample + c_begin;
  const int tid = threadIdx.x;
  constexpr int U = kAChunk / kPacket / kAThreads;   // 4
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;   // <c, u>, ||u||^2 (NS == 2); ||u||^2, <u, c>, ||c||^2 (NS == 3)
  auto term = [&](float c, float u) {
    if constexpr (NS == 2) {
      s0 += (double)c * (double)u;
      s1 += (double)u * (double)u;
    } else {
      s0 += (double)u * (double)u;
      s1 += (double)u * (double)c;
      s2 += (double)c * (double)c;
    }
  };
  // element (u, i) of this thread is chunk element (u*kAThreads + tid)*8 + i on both paths, as in k_apg_partial
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const uint32_t pk = u * kAThreads + tid;
    if (VEC) {
      if (pk * kPacket < cnt) {
        const size_t e = e0 + (size_t)pk * kPacket;
        Raw<TE> rc, ru;
        ldg_pk(rc, static_cast<const TE*>(p.ec) + e);
        ldg_pk(ru, static_cast<const TE*>(p.eu) + e);
        float fc[8], fu[8];
        unpack(rc, fc);
        unpack(ru, fu);
#pragma unroll
        for (int i = 0; i < 8; ++i) term(fc[i], fu[i]);
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t j = pk * kPacket + i;
        if (j < cnt) term(load_any(p.ec, p.model_dtype, e0 + j), load_any(p.eu, p.model_dtype, e0 + j));
      }
    }
  }
  s0 = apg_cta_sum(s0, warp_part);
  s1 = apg_cta_sum(s1, warp_part);
  if constexpr (NS == 3) s2 = apg_cta_sum(s2, warp_part);
  if (tid == 0) {
    double* o = p.partial + (size_t)blockIdx.x * NS;
    o[0] = s0; o[1] = s1;
    if constexpr (NS == 3) o[2] = s2;
  }
}

__global__ void __launch_bounds__(kAThreads) k_cfgzero_final(const __grid_constant__ ZParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kAThreads + threadIdx.x;
  if (b >= p.n_samples) return;
  const double* part = p.partial + b * p.chunks * 2;
  double scu = 0.0, suu = 0.0;
  for (uint32_t c = 0; c < p.chunks; ++c) {
    scu += part[c * 2];
    suu += part[c * 2 + 1];
  }
  p.s_out[b] = (float)(scu / (suu + 1e-8));   // diffusers' cfg_zero_star_scale epsilon
}

// The words of sample b from its merged sums, in fp64 with each op rounded. (p, q) is the top eigenvector of the Gram
// matrix [[A, B], [B, C]], taken from the row without cancellation (h <= 0: row 1, else row 2); with the eigen identity
// the projection <u, v1>*v1 is (p*p*u + p*q*c)/(p*p + q*q). n2 == 0 (A == C and B == 0: no unique top direction, both
// outputs zero included) gives (1, 0), plain CFG; a sum that is not finite gives NaN words.
__global__ void __launch_bounds__(kAThreads) k_tcfg_final(const __grid_constant__ ZParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kAThreads + threadIdx.x;
  if (b >= p.n_samples) return;
  const double* part = p.partial + b * p.chunks * 3;
  double A = 0.0, B = 0.0, C = 0.0;
  for (uint32_t c = 0; c < p.chunks; ++c) {
    A += part[c * 3];
    B += part[c * 3 + 1];
    C += part[c * 3 + 2];
  }
  float wu, wc;
  if (!(isfinite(A) && isfinite(B) && isfinite(C))) {
    wu = wc = __int_as_float(0x7fffffff);
  } else {
    const double h = 0.5 * (A - C);
    const double r = sqrt(h * h + B * B);
    double pv, qv;
    if (C >= A) { pv = B; qv = (-h) + r; }
    else        { pv = h + r; qv = B; }
    const double pp = pv * pv;
    const double n2 = pp + qv * qv;
    if (n2 == 0.0) { wu = 1.f; wc = 0.f; }
    else { wu = (float)(pp / n2); wc = (float)((pv * qv) / n2); }
  }
  p.s_out[2 * b] = wu;
  p.s_out[2 * b + 1] = wc;
}

static size_t zpass_workspace_bytes(uint64_t n_samples, uint64_t per_sample, int ns) {
  if (per_sample == 0 || n_samples == 0) return 0;
  const uint64_t chunks = (per_sample + kAChunk - 1) / kAChunk;
  return (size_t)(n_samples * chunks) * ns * sizeof(double);
}
size_t cfgzero_workspace_bytes(uint64_t n_samples, uint64_t per_sample) {
  return zpass_workspace_bytes(n_samples, per_sample, 2);
}
size_t tcfg_workspace_bytes(uint64_t n_samples, uint64_t per_sample) {
  return zpass_workspace_bytes(n_samples, per_sample, 3);
}

// the sums pass over both halves, then `final` per sample: two launches, no allocation, no sync
template <int NS>
static int launch_zpass(void (*final)(const ZParams), const char* what, float* s_out, const void* ec, const void* eu,
                        int model_dtype, uint64_t per_sample, uint64_t n, void* ws, size_t ws_bytes,
                        cudaStream_t stream) {
  ZParams p;
  memset(&p, 0, sizeof(p));
  p.ec = ec; p.eu = eu; p.s_out = s_out; p.model_dtype = model_dtype;
  p.per_sample = per_sample; p.n_samples = n / per_sample;
  p.chunks = (uint32_t)((per_sample + kAChunk - 1) / kAChunk);
  p.partial = static_cast<double*>(ws);
  if (ws == nullptr || ws_bytes < zpass_workspace_bytes(p.n_samples, per_sample, NS) ||
      (reinterpret_cast<uintptr_t>(ws) & 7)) {
    set_error("%s: workspace too small or not 8-byte aligned", what);
    return DPM_ERR_ARG;
  }
  if (p.n_samples * p.chunks > 0x7fffffffull) { set_error("%s: too many chunks", what); return DPM_ERR_UNSUPPORTED; }
  const uintptr_t am = model_dtype == DPM_F32 ? 31 : 15;
  const bool vec = per_sample % kPacket == 0 && (reinterpret_cast<uintptr_t>(ec) & am) == 0 &&
                   (reinterpret_cast<uintptr_t>(eu) & am) == 0;
  typedef void (*ZKernel)(const ZParams);
  ZKernel k = k_cfgzero_partial<float, false, NS>;   // any dtype, alignment or sample size
  if (vec) {
    if (model_dtype == DPM_F32) k = k_cfgzero_partial<float, true, NS>;
    else if (model_dtype == DPM_BF16) k = k_cfgzero_partial<__nv_bfloat16, true, NS>;
    else if (model_dtype == DPM_F16) k = k_cfgzero_partial<__half, true, NS>;
  }
  k<<<(unsigned)(p.n_samples * p.chunks), kAThreads, 0, stream>>>(p);
  final<<<(unsigned)((p.n_samples + kAThreads - 1) / kAThreads), kAThreads, 0, stream>>>(p);
  count_launch();
  count_launch();
  return DPM_OK;
}

int launch_cfgzero_scale(float* s_out, const void* ec, const void* eu, int model_dtype, uint64_t per_sample,
                         uint64_t n, void* ws, size_t ws_bytes, cudaStream_t stream) {
  return launch_zpass<2>(k_cfgzero_final, "cfg-zero* scale", s_out, ec, eu, model_dtype, per_sample, n, ws, ws_bytes,
                         stream);
}

int launch_tcfg_words(float* w_out, const void* ec, const void* eu, int model_dtype, uint64_t per_sample, uint64_t n,
                      void* ws, size_t ws_bytes, cudaStream_t stream) {
  return launch_zpass<3>(k_tcfg_final, "tcfg words", w_out, ec, eu, model_dtype, per_sample, n, ws, ws_bytes, stream);
}

// ---- Perp-Neg (dpm_perpneg_words; Armandpour, Sadeghian, Zheng, Sadeghian and Zhou, arXiv:2304.04968) -------------
// The K-way sibling of the CFG-Zero* pass: over u = e_uncond and e_1..e_K, d_k = e_k - u in fp64 and the K fp64 sums
// N = ||d_1||^2, P_k = <d_k, d_1> (k = 2..K), in k_cfgzero_partial's chunking, thread ownership, warp butterflies and
// chunk merge. k_perpneg_final then folds the sums with the host scales into one word per sample,
// w_1 = fl32(s_1 - s_2*c_2 - ... - s_K*c_K), c_k = P_k/N (0 when N == 0), which dpm_step_multi_masked reads as condition
// 1's period-1 weight map. Algorithmic bytes: (K+1)*s_model per element. (This file builds with -fmad=false: no
// product below is contracted into an fma.)
constexpr int kPNMax = 4;   // DPM_MAX_CONDITIONS

struct PNParams {
  const void* eu;
  const void* ec[kPNMax];
  double* partial;       // [n_samples * chunks][K]: N, P_2 .. P_K
  float* w_out;          // [n_samples]
  uint64_t per_sample;
  uint64_t n_samples;
  uint32_t chunks;
  int32_t model_dtype;
  int32_t n_cond;
  float scales[kPNMax];  // fl32(s_1) .. fl32(s_K)
};

// VEC: per_sample % 8 == 0 and all K+1 blocks aligned, TE their type. Otherwise element-wise (load_any).
template <typename TE, bool VEC, int K>
__global__ void __launch_bounds__(kAThreads) k_perpneg_partial(const __grid_constant__ PNParams p) {
  static_assert(K >= 2 && K <= kPNMax, "two to four conditions");
  __shared__ double warp_part[kAThreads / 32];
  const uint64_t sample = blockIdx.x / p.chunks;
  const uint32_t chunk = blockIdx.x % p.chunks;
  const uint64_t c_begin = (uint64_t)chunk * kAChunk;
  const uint64_t c_end = c_begin + kAChunk < p.per_sample ? c_begin + kAChunk : p.per_sample;
  const uint32_t cnt = (uint32_t)(c_end - c_begin);
  const size_t e0 = sample * p.per_sample + c_begin;
  const int tid = threadIdx.x;
  constexpr int U = kAChunk / kPacket / kAThreads;   // 4
  double s[K];   // N, P_2 .. P_K
#pragma unroll
  for (int k = 0; k < K; ++k) s[k] = 0.0;
  auto term = [&](float u, const float (&e)[K]) {
    const double d1 = (double)e[0] - (double)u;
    s[0] += d1 * d1;
#pragma unroll
    for (int k = 1; k < K; ++k) s[k] += ((double)e[k] - (double)u) * d1;
  };
  // element (u, i) of this thread is chunk element (u*kAThreads + tid)*8 + i on both paths, as in k_cfgzero_partial
#pragma unroll
  for (int it = 0; it < U; ++it) {
    const uint32_t pk = it * kAThreads + tid;
    if (VEC) {
      if (pk * kPacket < cnt) {
        const size_t e = e0 + (size_t)pk * kPacket;
        Raw<TE> ru, rc[K];
        ldg_pk(ru, static_cast<const TE*>(p.eu) + e);
#pragma unroll
        for (int k = 0; k < K; ++k) ldg_pk(rc[k], static_cast<const TE*>(p.ec[k]) + e);
        float fu[8], fc[K][8];
        unpack(ru, fu);
#pragma unroll
        for (int k = 0; k < K; ++k) unpack(rc[k], fc[k]);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float ev[K];
#pragma unroll
          for (int k = 0; k < K; ++k) ev[k] = fc[k][i];
          term(fu[i], ev);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t j = pk * kPacket + i;
        if (j < cnt) {
          float ev[K];
#pragma unroll
          for (int k = 0; k < K; ++k) ev[k] = load_any(p.ec[k], p.model_dtype, e0 + j);
          term(load_any(p.eu, p.model_dtype, e0 + j), ev);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < K; ++k) s[k] = apg_cta_sum(s[k], warp_part);
  if (tid == 0) {
    double* o = p.partial + (size_t)blockIdx.x * K;
#pragma unroll
    for (int k = 0; k < K; ++k) o[k] = s[k];
  }
}

// The word of sample b from its merged sums, in fp64 left to right with each op rounded: t = s_1, then
// t = t - s_k*c_k for k = 2..K, rounded to fp32 once. A sum that is not finite gives k_tcfg_final's NaN.
__global__ void __launch_bounds__(kAThreads) k_perpneg_final(const __grid_constant__ PNParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kAThreads + threadIdx.x;
  if (b >= p.n_samples) return;
  const int K = p.n_cond;
  const double* part = p.partial + b * p.chunks * K;
  double s[kPNMax] = {0.0, 0.0, 0.0, 0.0};
  for (uint32_t c = 0; c < p.chunks; ++c) {
#pragma unroll
    for (int k = 0; k < kPNMax; ++k)
      if (k < K) s[k] += part[c * K + k];
  }
  bool finite = true;
#pragma unroll
  for (int k = 0; k < kPNMax; ++k)
    if (k < K) finite = finite && isfinite(s[k]);
  float w = __int_as_float(0x7fffffff);
  if (finite) {
    double t = (double)p.scales[0];
#pragma unroll
    for (int k = 1; k < kPNMax; ++k) {
      if (k < K) {
        const double ck = s[0] == 0.0 ? 0.0 : s[k] / s[0];
        t = t - (double)p.scales[k] * ck;
      }
    }
    w = (float)t;
  }
  p.w_out[b] = w;
}

size_t perpneg_workspace_bytes(uint64_t n_samples, uint64_t per_sample) {
  return zpass_workspace_bytes(n_samples, per_sample, kPNMax);
}

template <int K>
static void launch_perpneg_partial(const PNParams& p, bool vec, cudaStream_t stream) {
  typedef void (*PKernel)(const PNParams);
  PKernel k = k_perpneg_partial<float, false, K>;   // any dtype, alignment or sample size
  if (vec) {
    if (p.model_dtype == DPM_F32) k = k_perpneg_partial<float, true, K>;
    else if (p.model_dtype == DPM_BF16) k = k_perpneg_partial<__nv_bfloat16, true, K>;
    else if (p.model_dtype == DPM_F16) k = k_perpneg_partial<__half, true, K>;
  }
  k<<<(unsigned)(p.n_samples * p.chunks), kAThreads, 0, stream>>>(p);
}

// the sums pass over the K+1 blocks, then the word per sample: two launches, no allocation, no sync
int launch_perpneg_words(float* w_out, const void* eu, const void* const* ec, const float* scales, int n_cond,
                         int model_dtype, uint64_t per_sample, uint64_t n, void* ws, size_t ws_bytes,
                         cudaStream_t stream) {
  PNParams p;
  memset(&p, 0, sizeof(p));
  p.eu = eu; p.w_out = w_out; p.model_dtype = model_dtype; p.n_cond = n_cond;
  for (int k = 0; k < n_cond; ++k) { p.ec[k] = ec[k]; p.scales[k] = scales[k]; }
  p.per_sample = per_sample; p.n_samples = n / per_sample;
  p.chunks = (uint32_t)((per_sample + kAChunk - 1) / kAChunk);
  p.partial = static_cast<double*>(ws);
  if (ws == nullptr || ws_bytes < perpneg_workspace_bytes(p.n_samples, per_sample) ||
      (reinterpret_cast<uintptr_t>(ws) & 7)) {
    set_error("perpneg words: workspace too small or not 8-byte aligned");
    return DPM_ERR_ARG;
  }
  if (p.n_samples * p.chunks > 0x7fffffffull) { set_error("perpneg words: too many chunks"); return DPM_ERR_UNSUPPORTED; }
  const uintptr_t am = model_dtype == DPM_F32 ? 31 : 15;
  bool vec = per_sample % kPacket == 0 && (reinterpret_cast<uintptr_t>(eu) & am) == 0;
  for (int k = 0; k < n_cond; ++k) vec = vec && (reinterpret_cast<uintptr_t>(ec[k]) & am) == 0;
  if (n_cond == 2) launch_perpneg_partial<2>(p, vec, stream);
  else if (n_cond == 3) launch_perpneg_partial<3>(p, vec, stream);
  else launch_perpneg_partial<4>(p, vec, stream);
  k_perpneg_final<<<(unsigned)((p.n_samples + kAThreads - 1) / kAThreads), kAThreads, 0, stream>>>(p);
  count_launch();
  count_launch();
  return DPM_OK;
}

}  // namespace dpm
