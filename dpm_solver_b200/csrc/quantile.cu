// quantile.cu -- exact per-sample quantile of |x0| for dynamic thresholding
// (DPM_Solver.dynamic_thresholding_fn, dpm_solver_pytorch.py:416-423).
//
// torch.quantile(|x0|.reshape(B,-1), q, dim=1) sorts every sample. Here x0 is never materialised:
// it is recomputed from (x, eps[, eps_u]) with the same device function the update kernel uses, and
// the two adjacent order statistics are found by selection on the fp32 bit pattern of |x0|
// (monotone as uint32 for non-negative floats). They are combined with torch's CPU lerp
// (fma(w<0.5 ? w : w-1, hi-lo, w<0.5 ? lo : hi)) and floored with max_val (:423). Non-finite order statistics
// follow torch: an infinite one can make the lerp inf - inf = NaN, a NaN anywhere in the sample makes the result
// NaN, and the floor keeps a NaN (torch.maximum), so the whole sample then becomes NaN.
//
// Two implementations behind dpm_dynamic_threshold():
//
//  A. streaming pipeline (needs a caller-provided workspace; used for samples of >= 8192 elements)
//     k_q_pivots : one CTA per sample gathers 1024 evenly strided keys, sorts them and derives two
//                  pivot keys that bracket the target rank (4 sigma of the sample-rank + slack).
//     k_q_count  : the heavy pass, full occupancy, one read of the inputs at HBM rate: counts keys
//                  below the bracket and compacts the ~2 % of keys inside it into the workspace
//                  (block-local list, one global atomic pair per CTA).
//     k_q_finish : one CTA per sample; the exact counts prove whether both target ranks lie inside
//                  the bracket; if so an 11/11/10-bit radix select over the candidates finishes,
//                  else (ties, adversarial data, mid-range q) the CTA runs the radix select over
//                  the whole sample from global memory. Always exact.
//  B. cluster kernel (no workspace, small samples): one thread-block cluster per sample, keys parked
//     in shared memory, per-digit histograms merged with distributed-shared-memory atomics.
#include <cooperative_groups.h>
#include <math.h>
#include <stdlib.h>

#include "common.cuh"
#include "launch.cuh"

namespace cg = cooperative_groups;

namespace dpm {

constexpr int kQThreads = 512;      // cluster kernel
constexpr int kBins = 2048;
constexpr int kSamples = 1024;      // sample keys per sample (pivot kernel)
constexpr int kPThreads = 256;      // pivot / count / finish kernels
constexpr int kLocalCand = 2048;    // bracket keys one count-CTA may collect
constexpr int kQUnroll = 2;         // count kernel: packets per thread per chunk
constexpr int kQIters = 4;          // count kernel: consecutive chunks per CTA

struct QParams {
  uint64_t lo;        // floor(pos)
  uint32_t two;       // 1 if ceil(pos) != floor(pos)
  float w;            // pos - floor(pos)
  float max_val;
  uint32_t cap;       // cluster: key capacity per CTA (0 => not cached); pipeline: candidates per sample
  uint32_t slice;     // cluster: elements owned by one CTA; pipeline: chunks per sample
  int32_t margin;     // half width of the bracket in sample ranks
  float* s_out;
  uint32_t* work;     // pipeline workspace: [n_samples][8] header words, then [n_samples][cap] candidates
  uint64_t n_samples;
  uint32_t num_space; // pipeline: bracket keys are |numerator| patterns (plain eps -> x0 map, alpha > 0)
};
// header words per sample
enum { H_LO = 0, H_HI = 1, H_LT = 2, H_IN = 3, H_PATH = 4, H_ALO = 5, H_AHI = 6, H_NAN = 7, H_WORDS = 8 };
constexpr uint32_t kInfKey = 0x7f800000u;   // |x0| bit patterns above this are NaN: torch.quantile then returns NaN

struct Sel {
  uint32_t bin, cnt;
  uint64_t rank;
};

// Block-wide: find the bin of tot[0 .. THREADS*PER) that holds 0-based rank k; every thread returns
// the same answer.
template <int THREADS, int PER>
__device__ __forceinline__ Sel select_bin(const uint32_t* tot, uint64_t k, uint32_t* warp_sums, Sel* out) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  uint32_t h[PER], local = 0;
#pragma unroll
  for (int i = 0; i < PER; ++i) { h[i] = tot[tid * PER + i]; local += h[i]; }
  uint32_t incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_sums[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    uint32_t v = lane < THREADS / 32 ? warp_sums[lane] : 0, s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    if (lane < THREADS / 32) warp_sums[lane] = s - v;  // exclusive
  }
  __syncthreads();
  uint64_t excl = (uint64_t)warp_sums[wid] + (incl - local);
  if (k >= excl && k < excl + local) {
    uint64_t c = excl;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      if (k >= c && k < c + h[i]) { out->bin = tid * PER + i; out->cnt = h[i]; out->rank = k - c; }
      c += h[i];
    }
  }
  __syncthreads();
  Sel r = *out;
  __syncthreads();
  return r;
}

// keys of one packet: |x0| bit patterns, x0 from the same packet function the update kernels use
template <int NE, typename TE, typename TS>
__device__ __forceinline__ void keys_of_packet(const KParams& p, const Raw<TS>& rx, const Raw<TE>& rc,
                                               const Raw<TE>& ru, uint32_t (&k8)[8]) {
  float fx[8], fc[8], fu[8], fT[8];
  unpack(rx, fx);
  unpack(rc, fc);
#pragma unroll
  for (int i = 0; i < 8; ++i) fu[i] = 0.f;
  if (NE == 2) unpack(ru, fu);
  if (p.fast_div && p.param == DPM_PARAM_NOISE) {
    fast_model8<NE>(p, fx, fc, fu, false, 1.f, fT);
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) fT[i] = model_value<NE>(p, fx[i], fc[i], fu[i], 1.f, false);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) k8[i] = __float_as_uint(fabsf(fT[i]));
}
template <int NE>
__device__ __forceinline__ uint32_t key_of_element(const KParams& p, size_t g) {
  float xe = load_any(p.xe, p.state_dtype, g);
  float ec = load_any(p.ec, p.model_dtype, g);
  float eu = NE == 2 ? load_any(p.eu, p.model_dtype, g) : 0.f;
  return __float_as_uint(fabsf(model_value<NE>(p, xe, ec, eu, 1.f, false)));
}

__device__ __forceinline__ float finish_value(uint32_t key_lo, uint32_t key_hi, const QParams& qp) {
  const float a = __uint_as_float(key_lo), b = __uint_as_float(key_hi);
  const float d = b - a;
  // at::native::lerp, CPU vectorised path: fmadd(coeff, end - start, base)
  // an infinite order statistic gives inf - inf = NaN (both infinite, or lo finite with w >= 0.5) exactly as in
  // torch, and torch.maximum keeps it
  float s = qp.w < 0.5f ? fmaf(qp.w, d, a) : fmaf(qp.w - 1.f, d, b);
  return max_nan(s, qp.max_val);  // torch.maximum(s, max_val) :423
}

// =================================== A. streaming pipeline ======================================
template <int NE>
__global__ void __launch_bounds__(kPThreads) k_q_pivots(const __grid_constant__ KParams p,
                                                         const __grid_constant__ QParams qp) {
  __shared__ uint32_t samp[kSamples];
  const uint64_t sample = blockIdx.x;
  const size_t s_begin = sample * p.per_sample;
  // 256 evenly strided groups of 4 consecutive elements: one 16/32-byte DRAM access serves 4 keys
  // (a strided single-element gather moves a 128-byte line per key). Neighbouring elements of real
  // images are correlated, so the bracket margin is sized for ~kSamples/4 independent draws.
  for (int j = threadIdx.x; j < kSamples; j += kPThreads) {
    const uint64_t grp = j >> 2;
    uint64_t pos = (uint64_t)(((unsigned __int128)grp * p.per_sample) / (kSamples / 4));
    pos = (pos & ~(uint64_t)3) + (j & 3);
    if (pos >= p.per_sample) pos = p.per_sample - 1;
    samp[j] = key_of_element<NE>(p, s_begin + pos);
  }
  __syncthreads();
  // only two order statistics of the sample are needed: 11/11/10-bit radix select in shared memory
  // (a full bitonic sort of the 1024 keys cost 10x the instructions and made this kernel issue-bound)
  __shared__ uint32_t hist[kBins];
  __shared__ __align__(16) uint32_t ctrl[32];
  __shared__ uint32_t s_piv[2];
  const int64_t ps_rank = (int64_t)(((unsigned __int128)qp.lo * kSamples) / p.per_sample);
  const int64_t want[2] = {ps_rank - qp.margin, ps_rank + qp.margin + 1};
#pragma unroll 1
  for (int which = 0; which < 2; ++which) {
    if (want[which] < 0 || want[which] >= kSamples) {
      if (threadIdx.x == 0) s_piv[which] = which == 0 ? 0u : 0xffffffffu;
      continue;
    }
    uint64_t rank = (uint64_t)want[which];
    uint32_t prefix = 0;
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {
      for (int i = threadIdx.x; i < kBins; i += kPThreads) hist[i] = 0;
      __syncthreads();
      for (int i = threadIdx.x; i < kSamples; i += kPThreads) {
        const uint32_t k = samp[i];
        if (pass == 0) atomicAdd(&hist[k >> 21], 1u);
        else if (pass == 1) { if ((k >> 21) == prefix) atomicAdd(&hist[(k >> 10) & 2047u], 1u); }
        else { if ((k >> 10) == prefix) atomicAdd(&hist[k & 1023u], 1u); }
      }
      __syncthreads();
      const Sel sc = select_bin<kPThreads, kBins / kPThreads>(hist, rank, ctrl, reinterpret_cast<Sel*>(ctrl + 20));
      rank = sc.rank;
      prefix = pass == 0 ? sc.bin : (pass == 1 ? ((prefix << 11) | sc.bin) : ((prefix << 10) | sc.bin));
    }
    if (threadIdx.x == 0) s_piv[which] = prefix;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t* h = qp.work + sample * H_WORDS;
    h[H_LO] = s_piv[0];
    h[H_HI] = s_piv[1];
    h[H_LT] = 0u;
    h[H_IN] = 0u;
    h[H_NAN] = 0u;
    // The same two thresholds in "numerator space". x0 = RN(num / alpha) with num = xe - sigma*eps
    // is a monotone non-decreasing function of |num|, so
    //   key(x0) <  lo  <=>  |num| <  A_lo,   A_lo = min{a : RN(a/alpha) >= float(lo)}
    //   key(x0) <= hi  <=>  |num| <= A_hi,   A_hi = max{a : RN(a/alpha) <= float(hi)}
    // and the count kernel can classify every element without dividing. Found exactly by walking
    // from the estimate lo*alpha to the boundary with nextafter steps (IEEE division here).
    const float al = p.alpha_e;
    float A_lo = 0.f, A_hi = __uint_as_float(0x7f800000u);
    const float L = __uint_as_float(h[H_LO]);
    if (h[H_LO] != 0u && al > 0.f) {
      float a = L * al;
      for (int it = 0; it < 64 && a > 0.f && (__uint_as_float(__float_as_uint(a) - 1u) / al) >= L; ++it)
        a = __uint_as_float(__float_as_uint(a) - 1u);
      for (int it = 0; it < 64 && (a / al) < L; ++it) a = __uint_as_float(__float_as_uint(a) + 1u);
      A_lo = a;
    }
    if (h[H_HI] != 0xffffffffu && al > 0.f) {
      const float Hh = __uint_as_float(h[H_HI]);
      float a = Hh * al;
      for (int it = 0; it < 64 && (__uint_as_float(__float_as_uint(a) + 1u) / al) <= Hh; ++it)
        a = __uint_as_float(__float_as_uint(a) + 1u);
      for (int it = 0; it < 64 && a > 0.f && (a / al) > Hh; ++it) a = __uint_as_float(__float_as_uint(a) - 1u);
      A_hi = a;
    }
    h[H_ALO] = __float_as_uint(A_lo);
    h[H_AHI] = __float_as_uint(A_hi);
  }
}

template <typename TE, typename TS, int NE, bool VEC, int U>
__global__ void __launch_bounds__(kPThreads) k_q_count(const __grid_constant__ KParams p,
                                                        const __grid_constant__ QParams qp) {
  constexpr int kChunk = U * kPacket * kPThreads;
  __shared__ uint32_t lcand[kLocalCand];
  __shared__ uint32_t s_n, s_lt, s_base;
  const uint32_t cps = qp.slice;                                   // CTAs per sample
  const uint64_t sample = blockIdx.x / cps;
  const uint32_t part = blockIdx.x % cps;
  uint32_t* hdr = qp.work + sample * H_WORDS;
  const bool num_space = qp.num_space != 0;
  const int tid = threadIdx.x;
  if (tid == 0) { s_n = 0; s_lt = 0; }
  __syncthreads();
  pdl_trigger();
  pdl_wait();      // the pivots kernel's header words (programmatic dependent launch: launch.cuh)
  const uint32_t lo_k = hdr[H_LO], hi_k = hdr[H_HI];
  const float A_lo = __uint_as_float(hdr[H_ALO]), A_hi = __uint_as_float(hdr[H_AHI]);

  uint32_t c_lt = 0, kmax = 0;   // kmax: largest |.| bit pattern seen (NaN detection, one integer max per element)
  // numerator space: 8 elements, ~8 instructions each and NO division at all: |num| -> |num / alpha| is
  // monotone for alpha > 0, so the bracket keys are collected as |num| bit patterns and k_q_finish
  // selects among them by rank and divides only the two order statistics it returns. One shared-memory
  // atomic per lane that holds bracket keys (about one lane in six), then predicated stores: with ~2 %
  // of the keys inside the bracket nearly every warp meets one per packet, so this path is hot.
  auto visit_num8 = [&](const float (&fx)[8], const float (&fc)[8], const float (&fu)[8]) {
    float a8[8];
    uint32_t mask = 0, n_ge = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float eps = (NE == 2) ? fu[i] + p.guidance * (fc[i] - fu[i]) : fc[i];   // :330
      a8[i] = fabsf(fx[i] - p.sigma_e * eps);                                        // |numerator| of :439
      kmax = max(kmax, __float_as_uint(a8[i]));
      const bool ge = a8[i] >= A_lo;
      n_ge += ge ? 1u : 0u;
      mask |= (ge && a8[i] <= A_hi) ? (1u << i) : 0u;
    }
    c_lt += 8u - n_ge;                                                               // NaN counts as "below", as before
    if (mask) {
      uint32_t pos = atomicAdd(&s_n, (uint32_t)__popc(mask));
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (mask & (1u << i)) {
          if (pos < kLocalCand) lcand[pos] = __float_as_uint(a8[i]);
          ++pos;
        }
      }
    }
  };
  // 8 keys at a time: branch-free counting, one (rarely taken) branch per packet for the bracket keys
  auto visit8 = [&](const uint32_t (&k8)[8]) {
    uint32_t mask = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const bool ge = k8[i] >= lo_k;
      kmax = max(kmax, k8[i]);
      c_lt += ge ? 0u : 1u;
      mask |= (ge && k8[i] <= hi_k) ? (1u << i) : 0u;
    }
    if (mask) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (mask & (1u << i)) {
          const uint32_t pos = atomicAdd(&s_n, 1u);
          if (pos < kLocalCand) lcand[pos] = k8[i];
        }
      }
    }
  };
  auto visit = [&](uint32_t k) {
    kmax = max(kmax, k);
    c_lt += k < lo_k ? 1u : 0u;
    if (k >= lo_k && k <= hi_k) {
      const uint32_t pos = atomicAdd(&s_n, 1u);
      if (pos < kLocalCand) lcand[pos] = k;
    }
  };
#pragma unroll 1
  for (uint32_t it = 0; it < kQIters; ++it) {
    const uint64_t c_begin = ((uint64_t)part * kQIters + it) * kChunk;
    if (c_begin >= p.per_sample) break;
    const uint64_t c_end = c_begin + kChunk < p.per_sample ? c_begin + kChunk : p.per_sample;
    const uint32_t cnt = (uint32_t)(c_end - c_begin);
    const size_t e0 = sample * p.per_sample + c_begin;
    if (VEC) {
      const TS* __restrict__ gxe = static_cast<const TS*>(p.xe);
      const TE* __restrict__ gec = static_cast<const TE*>(p.ec);
      const TE* __restrict__ geu = static_cast<const TE*>(p.eu);
      const uint32_t npk = cnt / kPacket;                          // per_sample % 8 == 0 here
      Raw<TS> rx[U];
      Raw<TE> rc[U], ru[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t pk = u * kPThreads + tid;
        if (pk < npk) {
          const size_t e = e0 + (size_t)pk * kPacket;
          ldg_pk(rx[u], gxe + e);
          ldg_pk(rc[u], gec + e);
          if (NE == 2) ldg_pk(ru[u], geu + e);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t pk = u * kPThreads + tid;
        if (pk < npk) {
          if (num_space) {
            float fx[8], fc[8], fu[8];
            unpack(rx[u], fx);
            unpack(rc[u], fc);
            if (NE == 2) unpack(ru[u], fu);
            visit_num8(fx, fc, fu);
          } else {
            uint32_t k8[8];
            keys_of_packet<NE>(p, rx[u], rc[u], ru[u], k8);
            visit8(k8);
          }
        }
      }
    } else {
      for (uint32_t i = tid; i < cnt; i += kPThreads) visit(key_of_element<NE>(p, e0 + i));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c_lt += __shfl_xor_sync(0xffffffffu, c_lt, o);
  if ((tid & 31) == 0 && c_lt) atomicAdd(&s_lt, c_lt);
  kmax = __reduce_max_sync(0xffffffffu, kmax);
  if ((tid & 31) == 0 && kmax > kInfKey) atomicOr(&hdr[H_NAN], 1u);
  __syncthreads();
  const uint32_t n_local = s_n;
  if (tid == 0) {
    if (s_lt) atomicAdd(&hdr[H_LT], s_lt);
    s_base = n_local ? atomicAdd(&hdr[H_IN], n_local) : 0u;        // H_IN counts every bracket key, stored or not
  }
  __syncthreads();
  if (n_local && n_local <= kLocalCand) {
    const uint32_t base = s_base;
    if ((uint64_t)base + n_local <= qp.cap) {
      uint32_t* cand = qp.work + qp.n_samples * H_WORDS + sample * (uint64_t)qp.cap;
      for (uint32_t i = tid; i < n_local; i += kPThreads) cand[base + i] = lcand[i];
    }
  } else if (n_local > kLocalCand && tid == 0) {
    atomicAdd(&hdr[H_IN], 0x40000000u);                            // poison: forces the exact fallback
  }
}

template <int NE>
__global__ void __launch_bounds__(kPThreads) k_q_finish(const __grid_constant__ KParams p,
                                                         const __grid_constant__ QParams qp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* cand = reinterpret_cast<uint32_t*>(smem_raw);          // [cap]: candidates staged once (3 passes read them)
  __shared__ uint32_t hist[kBins];
  __shared__ __align__(16) uint32_t ctrl[32];
  uint32_t* warp_sums = ctrl;
  uint32_t* min_slot = ctrl + 16;
  Sel* sel = reinterpret_cast<Sel*>(ctrl + 20);
  const uint64_t sample = blockIdx.x;
  const int tid = threadIdx.x;
  uint32_t* hdr = qp.work + sample * H_WORDS;
  pdl_trigger();
  pdl_wait();      // the count kernel's counters and candidates
  const uint64_t C_lt = hdr[H_LT], C_in = hdr[H_IN];
  const bool bracket_ok = C_in <= qp.cap && qp.lo >= C_lt && (qp.lo + qp.two) < C_lt + C_in;
  if (tid == 0) {
    *min_slot = 0xffffffffu;
    hdr[H_PATH] = bracket_ok ? 1u : 2u;   // diagnostics: which path finished this sample
  }

  uint64_t m;        // number of keys the select runs over
  uint64_t rank;
  const size_t s_begin = sample * p.per_sample;
  const uint32_t* gc = qp.work + qp.n_samples * H_WORDS + sample * (uint64_t)qp.cap;
  const bool staged = bracket_ok && qp.slice != 0 && C_in <= qp.cap;   // qp.slice reused: 1 = shared-memory staging fits
  if (bracket_ok) {
    if (staged)
      for (uint32_t i = tid; i < C_in; i += kPThreads) cand[i] = gc[i];
    m = C_in;
    rank = qp.lo - C_lt;
  } else {
    m = p.per_sample;                                              // exact fallback over the whole sample
    rank = qp.lo;
  }
  auto key_at = [&](uint64_t i) -> uint32_t {
    return bracket_ok ? (staged ? cand[i] : __ldcg(gc + i)) : key_of_element<NE>(p, s_begin + i);
  };
  __syncthreads();

  uint32_t prefix = 0;
  Sel sc;
#pragma unroll 1
  for (int pass = 0; pass < 3; ++pass) {
    for (int i = tid; i < kBins; i += kPThreads) hist[i] = 0;
    __syncthreads();
    for (uint64_t i = tid; i < m; i += kPThreads) {
      const uint32_t k = key_at(i);
      if (pass == 0) atomicAdd(&hist[k >> 21], 1u);
      else if (pass == 1) { if ((k >> 21) == prefix) atomicAdd(&hist[(k >> 10) & 2047u], 1u); }
      else { if ((k >> 10) == prefix) atomicAdd(&hist[k & 1023u], 1u); }
    }
    __syncthreads();
    sc = select_bin<kPThreads, kBins / kPThreads>(hist, rank, warp_sums, sel);
    rank = sc.rank;
    prefix = pass == 0 ? sc.bin : (pass == 1 ? ((prefix << 11) | sc.bin) : ((prefix << 10) | sc.bin));
  }
  const uint32_t key_lo = prefix;
  uint32_t key_hi = key_lo;
  if (qp.two && (sc.rank + 1 >= sc.cnt)) {                         // upper neighbour is the next larger key
    uint32_t mn = 0xffffffffu;
    for (uint64_t i = tid; i < m; i += kPThreads) {
      const uint32_t k = key_at(i);
      if (k > key_lo && k < mn) mn = k;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    if ((tid & 31) == 0 && mn != 0xffffffffu) atomicMin(min_slot, mn);
    __syncthreads();
    key_hi = *min_slot;
  }
  if (tid == 0) {
    uint32_t k_lo = key_lo, k_hi = key_hi;
    if (bracket_ok && qp.num_space) {
      // the candidates were |numerator| bit patterns (k_q_count): the order statistics of |x0| are the
      // IEEE quotients of the selected numerators (monotone map, alpha > 0)
      k_lo = __float_as_uint(__fdiv_rn(__uint_as_float(key_lo), p.alpha_e));
      k_hi = __float_as_uint(__fdiv_rn(__uint_as_float(key_hi), p.alpha_e));
    }
    // a NaN anywhere in the sample makes torch.quantile (and the maximum that follows, :422-423) return NaN
    qp.s_out[sample] = hdr[H_NAN] ? __uint_as_float(0x7fc00000u) : finish_value(k_lo, k_hi, qp);
  }
}

// =================================== B. cluster kernel ==========================================
template <typename TE, typename TS, int NE, bool VEC>
__global__ void __launch_bounds__(kQThreads)
    k_quantile_cluster(const __grid_constant__ KParams p, const __grid_constant__ QParams qp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* hist = reinterpret_cast<uint32_t*>(smem_raw);          // [kBins] local digit histogram
  uint32_t* total = hist + kBins;                                  // [3][kBins] cluster totals (rank 0)
  uint32_t* ctrl = total + 3 * kBins;                              // [64] warp sums, min slot, Sel
  uint32_t* keys = ctrl + 64;                                      // [cap]
  uint32_t* warp_sums = ctrl;                                      // 16 used
  uint32_t* min_slot = ctrl + 32;
  uint32_t* max_slot = ctrl + 33;                                  // largest key of the sample (NaN detection)
  Sel* sel = reinterpret_cast<Sel*>(ctrl + 40);

  cg::cluster_group cluster = cg::this_cluster();
  const uint32_t crank = cluster.block_rank();
  const uint32_t csize = cluster.num_blocks();
  const uint64_t sample = blockIdx.x / csize;
  const int tid = threadIdx.x;

  const uint64_t s_begin = sample * p.per_sample;                  // first element of the sample
  uint64_t c_begin = (uint64_t)crank * qp.slice;                   // slice inside the sample
  uint64_t c_end = c_begin + qp.slice;
  if (c_begin > p.per_sample) c_begin = p.per_sample;
  if (c_end > p.per_sample) c_end = p.per_sample;
  const uint32_t cnt = (uint32_t)(c_end - c_begin);

  for (int i = tid; i < kBins; i += kQThreads) hist[i] = 0;
  for (int i = tid; i < 3 * kBins; i += kQThreads) total[i] = 0;
  if (tid == 0) { *min_slot = 0xffffffffu; *max_slot = 0u; }
  uint32_t kmax = 0;
  __syncthreads();

  const TS* __restrict__ gxe = static_cast<const TS*>(p.xe);
  const TE* __restrict__ gec = static_cast<const TE*>(p.ec);
  const TE* __restrict__ geu = static_cast<const TE*>(p.eu);

  // key(i) for element i of this CTA's slice, recomputed from global memory
  auto key_scalar = [&](uint32_t i) -> uint32_t {
    const size_t g = s_begin + c_begin + i;
    float xe = load_any(p.xe, p.state_dtype, g);
    float ec = load_any(p.ec, p.model_dtype, g);
    float eu = NE == 2 ? load_any(p.eu, p.model_dtype, g) : 0.f;
    float v = model_value<NE>(p, xe, ec, eu, 1.f, false);
    return __float_as_uint(fabsf(v));
  };

  // ---- pass A: stream the slice once, stage keys, histogram of bits 31..21 ----
  if (VEC) {
    const uint32_t npk = cnt / kPacket;
    const size_t e0 = s_begin + c_begin;
    for (uint32_t pk0 = 0; pk0 < npk; pk0 += 2 * kQThreads) {
      Raw<TS> rx[2];
      Raw<TE> rc[2], ru[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint32_t pk = pk0 + u * kQThreads + tid;
        if (pk < npk) {
          const size_t e = e0 + (size_t)pk * kPacket;
          ldg_pk(rx[u], gxe + e);
          ldg_pk(rc[u], gec + e);
          if (NE == 2) ldg_pk(ru[u], geu + e);
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const uint32_t pk = pk0 + u * kQThreads + tid;
        if (pk < npk) {
          uint32_t k8[8];
          keys_of_packet<NE>(p, rx[u], rc[u], ru[u], k8);
#pragma unroll
          for (int i = 0; i < 8; ++i) { atomicAdd(&hist[k8[i] >> 21], 1u); kmax = max(kmax, k8[i]); }
          if (qp.cap) {
            uint4* dst = reinterpret_cast<uint4*>(keys + (size_t)pk * kPacket);
            dst[0] = make_uint4(k8[0], k8[1], k8[2], k8[3]);
            dst[1] = make_uint4(k8[4], k8[5], k8[6], k8[7]);
          }
        }
      }
    }
  } else {
    for (uint32_t i = tid; i < cnt; i += kQThreads) {
      uint32_t k = key_scalar(i);
      kmax = max(kmax, k);
      atomicAdd(&hist[k >> 21], 1u);
      if (qp.cap) keys[i] = k;
    }
  }
  auto key_at = [&](uint32_t i) -> uint32_t { return qp.cap ? keys[i] : key_scalar(i); };

  uint32_t* total0 = csize > 1 ? cluster.map_shared_rank(total, 0) : total;
  uint32_t* min0 = csize > 1 ? cluster.map_shared_rank(min_slot, 0) : min_slot;
  uint32_t* max0 = csize > 1 ? cluster.map_shared_rank(max_slot, 0) : max_slot;
  kmax = __reduce_max_sync(0xffffffffu, kmax);

  auto merge = [&](int pass, int nb) {
    __syncthreads();
    if (pass == 0 && csize > 1) cluster.sync();  // every CTA has zeroed its arrays
    if (pass == 0 && (tid & 31) == 0 && kmax > kInfKey) atomicMax(max0, kmax);
    for (int i = tid; i < nb; i += kQThreads) {
      uint32_t v = hist[i];
      if (v) atomicAdd(&total0[pass * kBins + i], v);
    }
    if (csize > 1) cluster.sync(); else __syncthreads();
  };

  merge(0, kBins);
  Sel sa = select_bin<kQThreads, kBins / kQThreads>(total0, qp.lo, warp_sums, sel);

  // ---- pass B: bits 20..10 among keys whose top digit matches ----
  for (int i = tid; i < kBins; i += kQThreads) hist[i] = 0;
  __syncthreads();
  for (uint32_t i = tid; i < cnt; i += kQThreads) {
    uint32_t k = key_at(i);
    if ((k >> 21) == sa.bin) atomicAdd(&hist[(k >> 10) & 2047u], 1u);
  }
  merge(1, kBins);
  Sel sb = select_bin<kQThreads, kBins / kQThreads>(total0 + kBins, sa.rank, warp_sums, sel);
  const uint32_t prefix22 = (sa.bin << 11) | sb.bin;

  // ---- pass C: bits 9..0 ----
  for (int i = tid; i < kBins; i += kQThreads) hist[i] = 0;
  __syncthreads();
  for (uint32_t i = tid; i < cnt; i += kQThreads) {
    uint32_t k = key_at(i);
    if ((k >> 10) == prefix22) atomicAdd(&hist[k & 1023u], 1u);
  }
  merge(2, 1024);
  Sel sc = select_bin<kQThreads, kBins / kQThreads>(total0 + 2 * kBins, sb.rank, warp_sums, sel);
  const uint32_t key_lo = (prefix22 << 10) | sc.bin;

  // ---- upper neighbour ----
  uint32_t key_hi = key_lo;
  const bool need_next = qp.two && (sc.rank + 1 >= sc.cnt);  // uniform across the cluster
  if (need_next) {
    uint32_t m = 0xffffffffu;
    for (uint32_t i = tid; i < cnt; i += kQThreads) {
      uint32_t k = key_at(i);
      if (k > key_lo && k < m) m = k;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0 && m != 0xffffffffu) atomicMin(min0, m);
    if (csize > 1) cluster.sync(); else __syncthreads();
    key_hi = *min0;
  }
  if (crank == 0 && tid == 0) {
    float s = finish_value(key_lo, key_hi, qp);
    if (*max0 > kInfKey) s = __uint_as_float(0x7fc00000u);   // NaN in the sample: torch.quantile returns NaN
    qp.s_out[sample] = s;
  }
  if (csize > 1) cluster.sync();  // keep CTA 0's shared memory alive until every peer has read it
}


typedef void (*QKernel)(const KParams, const QParams);
struct QKernels {
  QKernel cluster, count;
};

static uint32_t pipeline_cap(uint64_t ps) {
  // the 4-sigma bracket of a 1024-key sample holds <= 2*(4*sqrt(1024*q(1-q))+3)+1 sample ranks; for
  // q = 0.995 that is < 2 % of the keys (one-sided: the bracket is clipped at the maximum)
  // the bracket itself is a random variable (its lower pivot is an order statistic of the sample):
  // measured on N(0,1) data at q = 0.995 it holds 1.2 - 5.2 % of the keys; 6.25 % + 2048 leaves > 4 sigma
  uint64_t cap = ps / 16 + 2048;
  if (cap > (1u << 20)) cap = 1u << 20;
  return (uint32_t)cap;
}

size_t quantile_workspace_bytes(uint64_t n_samples, uint64_t per_sample) {
  if (per_sample < 8192) return 0;
  return (size_t)n_samples * (H_WORDS + (size_t)pipeline_cap(per_sample)) * sizeof(uint32_t);
}

int launch_quantile(float* s_out, const KParams& p, uint64_t n_samples, float q, float max_val,
                    void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const int md = p.model_dtype, sd = p.state_dtype;
  const uint64_t ps = p.per_sample;
  bool vec = (ps % kPacket == 0);
  // packet path needs aligned bases (sample starts stay aligned because ps % 8 == 0)
  auto al = [](const void* ptr, int dt) { return (reinterpret_cast<uintptr_t>(ptr) & (dt == DPM_F32 ? 31 : 15)) == 0; };
  if (!al(p.xe, sd) || !al(p.ec, md) || (p.n_model == 2 && !al(p.eu, md))) vec = false;

  auto pick = [&](auto pair) -> QKernels {
    using TE = typename decltype(pair)::TE;
    using TS = typename decltype(pair)::TS;
    if (p.n_model == 2)
      return {vec ? k_quantile_cluster<TE, TS, 2, true> : k_quantile_cluster<TE, TS, 2, false>,
              vec ? k_q_count<TE, TS, 2, true, kQUnroll> : k_q_count<TE, TS, 2, false, kQUnroll>};
    return {vec ? k_quantile_cluster<TE, TS, 1, true> : k_quantile_cluster<TE, TS, 1, false>,
            vec ? k_q_count<TE, TS, 1, true, kQUnroll> : k_q_count<TE, TS, 1, false, kQUnroll>};
  };
  QKernels k = with_packet_pair(md, sd, pick);   // the step kernels' five pairs
  if (k.cluster == nullptr) {
    if (md == DPM_F32 && sd == DPM_BF16) {   // fp32 network output, 16-bit state
      k = pick(PacketPair<float, __nv_bfloat16>{});
    } else if (md == DPM_F32 && sd == DPM_F16) {
      k = pick(PacketPair<float, __half>{});
    } else if ((md == DPM_BF16 && sd == DPM_F16) || (md == DPM_F16 && sd == DPM_BF16)) {
      // two different 16-bit types have no packet instantiation: the VEC = false kernels read every operand
      // through load_any with the runtime dtypes (the template types are unused there)
      vec = false;
      k = pick(PacketPair<float, float>{});
    } else {
      set_error("dynamic threshold: unsupported dtype mix (model %d, state %d)", md, sd);
      return DPM_ERR_UNSUPPORTED;
    }
  }

  // torch.quantile rank arithmetic, in fp32: pos = fl(q * (n-1))
  const float pos = q * (float)(ps - 1);
  const float fl = floorf(pos);
  QParams qp;
  memset(&qp, 0, sizeof(qp));
  qp.lo = (uint64_t)fl;
  qp.two = ceilf(pos) != fl ? 1u : 0u;
  qp.w = pos - fl;
  qp.max_val = max_val;
  qp.s_out = s_out;
  qp.n_samples = n_samples;
  if (qp.lo >= ps) qp.lo = ps - 1;
  if (qp.lo + 1 >= ps) qp.two = 0;
  if (n_samples > 0x7fffffffull / 16) { set_error("too many samples"); return DPM_ERR_UNSUPPORTED; }
  cudaError_t e;

  // ---- A. streaming pipeline ----
  const char* force = getenv("DPM_QUANTILE_IMPL");
  const bool want_pipeline = !(force && force[0] == 'c');
  const size_t need = quantile_workspace_bytes(n_samples, ps);
  if (want_pipeline && need != 0 && workspace != nullptr && workspace_bytes >= need &&
      (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && ps < (1ull << 32)) {
    const double f = ps > 1 ? (double)qp.lo / (double)(ps - 1) : 0.0;
    qp.margin = (int32_t)(6.0 * sqrt((double)kSamples * f * (1.0 - f)) + 3.0);   // 4 sigma at ~kSamples/2 effective draws
    qp.cap = pipeline_cap(ps);
    const uint64_t per_cta = (uint64_t)kQUnroll * kPacket * kPThreads * kQIters;
    qp.slice = (uint32_t)((ps + per_cta - 1) / per_cta);
    qp.work = static_cast<uint32_t*>(workspace);
    // division-free classification and |numerator| candidates need the plain eps -> x0 map with a positive alpha
    qp.num_space = (vec && p.param == DPM_PARAM_NOISE && p.predict_x0 && p.alpha_e > 0.f) ? 1u : 0u;
    if (n_samples * qp.slice > 0x7fffffffull) { set_error("too many chunks"); return DPM_ERR_UNSUPPORTED; }
    QKernel kp = p.n_model == 2 ? k_q_pivots<2> : k_q_pivots<1>;
    QKernel kf = p.n_model == 2 ? k_q_finish<2> : k_q_finish<1>;
    kp<<<(unsigned)n_samples, kPThreads, 0, stream>>>(p, qp);
    e = launch_pdl(k.count, (unsigned)(n_samples * qp.slice), kPThreads, 0, stream, p, qp);
    if (e != cudaSuccess) return launch_error("quantile count launch failed", e);
    // finish: stage the candidates in shared memory when they fit next to 3 co-resident CTAs (else read L2)
    QParams qf = qp;
    const size_t fsmem = (size_t)qp.cap * sizeof(uint32_t);
    qf.slice = fsmem <= 64 * 1024 ? 1u : 0u;
    if (qf.slice) {
      int rc = ensure_max_smem(reinterpret_cast<const void*>(kf));
      if (rc != 0) return rc;
    }
    e = launch_pdl(kf, (unsigned)n_samples, kPThreads, qf.slice ? fsmem : 0, stream, p, qf);
    if (e != cudaSuccess) return launch_error("quantile finish launch failed", e);
    count_launch();
    count_launch();
    count_launch();
    return DPM_OK;
  }

  // ---- B. cluster kernel ----
  // cluster size: smallest power of two whose per-CTA slice fits the shared-memory key cache
  const size_t fixed = (size_t)(kBins + 3 * kBins + 64) * sizeof(uint32_t);
  const size_t budget = (size_t)max_smem_optin();
  const uint64_t cap_max = budget > fixed ? (budget - fixed) / sizeof(uint32_t) : 0;
  int cs = 1;
  auto slice_for = [&](int c) {
    uint64_t s = (ps + c - 1) / c;
    return (s + kPacket - 1) / kPacket * kPacket;
  };
  while (cs < 16 && slice_for(cs) > cap_max) cs *= 2;
  uint64_t slice = slice_for(cs);
  // prefer >= 2 CTAs' worth of parallelism per sample when samples are few and large
  while (cs < 8 && n_samples * cs < (uint64_t)sm_count() && slice_for(cs * 2) >= 4096) { cs *= 2; slice = slice_for(cs); }
  uint32_t cap = slice <= cap_max ? (uint32_t)slice : 0;  // 0: recompute keys from L2/HBM each pass
  if (cap == 0) { cs = 8; slice = slice_for(cs); }
  qp.cap = cap;
  qp.slice = (uint32_t)slice;
  if (slice > 0xffffffffull) { set_error("per_sample too large"); return DPM_ERR_UNSUPPORTED; }

  const size_t smem = fixed + (size_t)cap * sizeof(uint32_t);
  int rc = ensure_max_smem(reinterpret_cast<const void*>(k.cluster), /*nonportable_cluster=*/true);
  if (rc != 0) return rc;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(n_samples * cs), 1, 1);
  cfg.blockDim = dim3(kQThreads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, k.cluster, p, qp);
  if (e != cudaSuccess) return launch_error("quantile launch failed", e);
  count_launch();
  return DPM_OK;
}

}  // namespace dpm
