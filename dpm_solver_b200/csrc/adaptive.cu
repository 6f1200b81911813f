// adaptive.cu -- error estimate of the adaptive step-size solver (dpm_solver_adaptive,
// dpm_solver_pytorch.py:999-1001):
//   delta = max(atol, rtol * max(|x_lower|, |x_prev|))
//   E     = max_b sqrt( mean_b( ((x_higher - x_lower) / delta)^2 ) )
// The reference spends 9 full-tensor eager ops on it; here one streaming pass produces per-chunk
// partial sums (fixed chunking and a fixed reduction tree: deterministic, unlike atomics) and a
// one-CTA epilogue folds them per sample in index order, takes sqrt(mean) and the batch maximum.
// Algorithmic bytes: 3*s per element read, one float written.
// The per-sample ratio of guidance rescale (below) reuses the same chunk -> CTA mapping.
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kEThreads = 256;
constexpr int kEChunk = 8192;   // elements per CTA

struct EParams {
  const void* xh;
  const void* xl;
  const void* xp;
  float* partial;        // [n_samples * chunks]
  float* out;            // [1]
  uint64_t per_sample;
  uint64_t n_samples;
  uint32_t chunks;       // per sample
  int32_t dtype;
  float atol, rtol;
};

template <typename T, bool VEC>
__global__ void __launch_bounds__(kEThreads) k_err_partial(const __grid_constant__ EParams p) {
  __shared__ float warp_sum[kEThreads / 32];
  const uint64_t sample = blockIdx.x / p.chunks;
  const uint32_t chunk = blockIdx.x % p.chunks;
  const uint64_t c_begin = (uint64_t)chunk * kEChunk;
  const uint64_t c_end = c_begin + kEChunk < p.per_sample ? c_begin + kEChunk : p.per_sample;
  const uint32_t cnt = (uint32_t)(c_end - c_begin);
  const size_t e0 = sample * p.per_sample + c_begin;
  const int tid = threadIdx.x;
  float acc = 0.f;
  auto term = [&](float h, float l, float q) {
    const float delta = max_nan(p.atol, p.rtol * max_nan(fabsf(l), fabsf(q)));   // :999
    const float v = (h - l) / delta;                                           // :1001
    acc += v * v;
  };
  if (VEC) {
    const T* gh = static_cast<const T*>(p.xh);
    const T* gl = static_cast<const T*>(p.xl);
    const T* gp = static_cast<const T*>(p.xp);
    const uint32_t npk = cnt / kPacket;
    constexpr int U = kEChunk / kPacket / kEThreads;   // 4
    Raw<T> rh[U], rl[U], rp[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t pk = u * kEThreads + tid;
      if (pk < npk) {
        const size_t e = e0 + (size_t)pk * kPacket;
        ldg_pk(rh[u], gh + e);
        ldg_pk(rl[u], gl + e);
        ldg_pk(rp[u], gp + e);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t pk = u * kEThreads + tid;
      if (pk < npk) {
        float fh[8], fl[8], fp[8];
        unpack(rh[u], fh);
        unpack(rl[u], fl);
        unpack(rp[u], fp);
#pragma unroll
        for (int i = 0; i < 8; ++i) term(fh[i], fl[i], fp[i]);
      }
    }
  } else {
    for (uint32_t i = tid; i < cnt; i += kEThreads)
      term(load_any(p.xh, p.dtype, e0 + i), load_any(p.xl, p.dtype, e0 + i), load_any(p.xp, p.dtype, e0 + i));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((tid & 31) == 0) warp_sum[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kEThreads / 32; ++w) s += warp_sum[w];
    p.partial[blockIdx.x] = s;
  }
}

__global__ void __launch_bounds__(kEThreads) k_err_final(const __grid_constant__ EParams p) {
  __shared__ float best[kEThreads];
  float mx = 0.f;
  for (uint64_t b = threadIdx.x; b < p.n_samples; b += kEThreads) {
    double s = 0.0;
    for (uint32_t c = 0; c < p.chunks; ++c) s += (double)p.partial[b * p.chunks + c];
    const float e = sqrtf((float)(s / (double)p.per_sample));   // norm_fn :1000
    mx = max_nan(mx, e);   // a NaN error norm must reach the controller (reference: torch .max())
  }
  best[threadIdx.x] = mx;
  __syncthreads();
  for (int o = kEThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) best[threadIdx.x] = max_nan(best[threadIdx.x], best[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) p.out[0] = best[0];   // .max() :1001
}

size_t adaptive_workspace_bytes(uint64_t n, uint64_t per_sample) {
  if (per_sample == 0 || n == 0) return 0;
  const uint64_t chunks = (per_sample + kEChunk - 1) / kEChunk;
  return (size_t)((n / per_sample) * chunks) * sizeof(float);
}

int launch_adaptive_error(float* out, const void* xh, const void* xl, const void* xp, float atol, float rtol,
                          uint64_t per_sample, uint64_t n, int dtype, void* ws, size_t ws_bytes, cudaStream_t stream) {
  EParams p;
  p.xh = xh; p.xl = xl; p.xp = xp; p.out = out; p.per_sample = per_sample; p.n_samples = n / per_sample;
  p.chunks = (uint32_t)((per_sample + kEChunk - 1) / kEChunk);
  p.dtype = dtype; p.atol = atol; p.rtol = rtol;
  p.partial = static_cast<float*>(ws);
  if (ws == nullptr || ws_bytes < adaptive_workspace_bytes(n, per_sample)) { set_error("adaptive error: workspace too small"); return DPM_ERR_ARG; }
  if (p.n_samples * p.chunks > 0x7fffffffull) { set_error("adaptive error: too many chunks"); return DPM_ERR_UNSUPPORTED; }
  auto al = [&](const void* q) { return (reinterpret_cast<uintptr_t>(q) & (dtype == DPM_F32 ? 31 : 15)) == 0; };
  const bool vec = per_sample % kPacket == 0 && al(xh) && al(xl) && al(xp);
  const unsigned grid = (unsigned)(p.n_samples * p.chunks);
  typedef void (*EKernel)(const EParams);
  EKernel k = with_packet_pair(dtype, dtype, [&](auto pair) -> EKernel {
    using T = typename decltype(pair)::TS;
    return vec ? k_err_partial<T, true> : k_err_partial<T, false>;
  });
  k<<<grid, kEThreads, 0, stream>>>(p);
  k_err_final<<<1, kEThreads, 0, stream>>>(p);
  count_launch();
  count_launch();
  return DPM_OK;
}

// ---- guidance rescale ratio (dpm_cfg_rescale_ratio) ------------------------------------------------------
//   g = out_u + s*(out_c - out_u)   (the step kernels' combine, :330)
//   r[b] = fl32(std(out_c[b])) / fl32(std(g[b])),  std unbiased, in fp64
// Same chunking as the error estimate: CTA (b, c) holds chunk c of sample b in registers, takes its fp64 mean
// (first pass) and the sum of squared deviations from that mean (second pass, exact for any mean/std ratio an
// fp32 sample can have); the final kernel merges the chunks of a sample in chunk order (Chan et al.'s pairwise
// update). Every thread owns the same elements on the vector and the element-wise path and all sums run in a fixed
// order, so r[b] depends on sample b's values only -- not on the batch, the sample's position or the alignment.
struct RParams {
  const void* ec;
  const void* eu;
  double* partial;       // [n_samples * chunks][4]: mean_c, M2_c, mean_g, M2_g
  float* ratio;          // [n_samples]
  uint64_t per_sample;
  uint64_t n_samples;
  uint32_t chunks;       // per sample
  int32_t dtype;
  float guidance;
  const float* gscale;   // per-sample scales [n_samples] in place of `guidance` (<PG = true> only)
};

// deterministic CTA sum of one double per thread (butterfly within the warps, then the warps in order)
__device__ __forceinline__ double cta_sum(double v, double* warp_part) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();   // warp_part may still be read from the previous call
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < kEThreads / 32; ++w) s += warp_part[w];
  return s;
}

// the scale of the combine: the launch's, or with PG sample b's
template <bool PG>
__device__ __forceinline__ float ratio_scale(const RParams& p, uint64_t sample) {
  if constexpr (PG) return __ldg(p.gscale + sample);
  else return p.guidance;
}

// PG: per-sample guidance (dpm_cfg_rescale_ratio_guided): g = out_u + s_b*(out_c - out_u) with the sample's scale
template <typename T, bool VEC, bool PG = false>
__global__ void __launch_bounds__(kEThreads) k_cfg_ratio_partial(const __grid_constant__ RParams p) {
  __shared__ double warp_part[2][kEThreads / 32];
  const uint64_t sample = blockIdx.x / p.chunks;
  const uint32_t chunk = blockIdx.x % p.chunks;
  const uint64_t c_begin = (uint64_t)chunk * kEChunk;
  const uint64_t c_end = c_begin + kEChunk < p.per_sample ? c_begin + kEChunk : p.per_sample;
  const uint32_t cnt = (uint32_t)(c_end - c_begin);
  const size_t e0 = sample * p.per_sample + c_begin;
  const int tid = threadIdx.x;
  constexpr int U = kEChunk / kPacket / kEThreads;   // 4
  // element (u, i) of this thread is chunk element (u*kEThreads + tid)*8 + i on both paths
  float fc[U][8], fg[U][8];
  if (VEC) {   // per_sample % 8 == 0: every packet of the chunk is full
    const T* gc = static_cast<const T*>(p.ec);
    const T* gu = static_cast<const T*>(p.eu);
    Raw<T> rc[U], ru[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t pk = u * kEThreads + tid;
      if (pk * kPacket < cnt) {
        ldg_pk(rc[u], gc + e0 + (size_t)pk * kPacket);
        ldg_pk(ru[u], gu + e0 + (size_t)pk * kPacket);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t pk = u * kEThreads + tid;
      if (pk * kPacket < cnt) {
        float fu[8];
        unpack(rc[u], fc[u]);
        unpack(ru[u], fu);
#pragma unroll
        for (int i = 0; i < 8; ++i) fg[u][i] = fu[i] + ratio_scale<PG>(p, sample) * (fc[u][i] - fu[i]);   // :330
      }
    }
  } else {
#pragma unroll
    for (int u = 0; u < U; ++u) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t k = (u * kEThreads + tid) * kPacket + i;
        if (k < cnt) {
          const float c = load_any(p.ec, p.dtype, e0 + k), uu = load_any(p.eu, p.dtype, e0 + k);
          fc[u][i] = c;
          fg[u][i] = uu + ratio_scale<PG>(p, sample) * (c - uu);   // :330
        }
      }
    }
  }
  auto live = [&](int u, int i) { return (uint32_t)((u * kEThreads + tid) * kPacket + i) < cnt; };
  double sc = 0.0, sg = 0.0;
#pragma unroll
  for (int u = 0; u < U; ++u) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (live(u, i)) {
        sc += (double)fc[u][i];
        sg += (double)fg[u][i];
      }
    }
  }
  const double mc = cta_sum(sc, warp_part[0]) / (double)cnt;
  const double mg = cta_sum(sg, warp_part[1]) / (double)cnt;
  double qc = 0.0, qg = 0.0;
#pragma unroll
  for (int u = 0; u < U; ++u) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (live(u, i)) {
        const double dc = (double)fc[u][i] - mc, dg = (double)fg[u][i] - mg;
        qc += dc * dc;
        qg += dg * dg;
      }
    }
  }
  qc = cta_sum(qc, warp_part[0]);
  qg = cta_sum(qg, warp_part[1]);
  if (tid == 0) {
    double* o = p.partial + (size_t)blockIdx.x * 4;
    o[0] = mc; o[1] = qc; o[2] = mg; o[3] = qg;
  }
}

__global__ void __launch_bounds__(kEThreads) k_cfg_ratio_final(const __grid_constant__ RParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kEThreads + threadIdx.x;
  if (b >= p.n_samples) return;
  const double* part = p.partial + b * p.chunks * 4;
  double n = 0.0, mc = 0.0, qc = 0.0, mg = 0.0, qg = 0.0;
  for (uint32_t c = 0; c < p.chunks; ++c) {
    const uint64_t c_begin = (uint64_t)c * kEChunk;
    const double nb = (double)((c_begin + kEChunk < p.per_sample ? c_begin + kEChunk : p.per_sample) - c_begin);
    const double* q = part + (size_t)c * 4;
    if (c == 0) {
      mc = q[0]; qc = q[1]; mg = q[2]; qg = q[3];
    } else {
      const double nab = n + nb, wb = nb / nab, wab = n * nb / nab;
      const double dc = q[0] - mc, dg = q[2] - mg;
      mc = mc + dc * wb;
      qc = (qc + q[1]) + dc * dc * wab;
      mg = mg + dg * wb;
      qg = (qg + q[3]) + dg * dg * wab;
    }
    n += nb;
  }
  // unbiased (torch.std's default correction): one sample gives 0/0 = NaN; each std is rounded to fp32 once
  const float std_c = (float)sqrt(qc / (n - 1.0));
  const float std_g = (float)sqrt(qg / (n - 1.0));
  p.ratio[b] = std_c / std_g;
}

size_t cfg_rescale_workspace_bytes(uint64_t n_samples, uint64_t per_sample) {
  if (per_sample == 0 || n_samples == 0) return 0;
  const uint64_t chunks = (per_sample + kEChunk - 1) / kEChunk;
  return (size_t)(n_samples * chunks) * 4 * sizeof(double);
}

int launch_cfg_rescale_ratio(float* ratio, const void* ec, const void* eu, float guidance, uint64_t per_sample,
                             uint64_t n, int dtype, void* ws, size_t ws_bytes, cudaStream_t stream,
                             const float* gscale) {
  RParams p;
  p.gscale = gscale;
  p.ec = ec; p.eu = eu; p.ratio = ratio; p.per_sample = per_sample; p.n_samples = n / per_sample;
  p.chunks = (uint32_t)((per_sample + kEChunk - 1) / kEChunk);
  p.dtype = dtype; p.guidance = guidance;
  p.partial = static_cast<double*>(ws);
  if (ws == nullptr || ws_bytes < cfg_rescale_workspace_bytes(p.n_samples, per_sample) ||
      (reinterpret_cast<uintptr_t>(ws) & 7)) {
    set_error("cfg rescale: workspace too small or not 8-byte aligned");
    return DPM_ERR_ARG;
  }
  if (p.n_samples * p.chunks > 0x7fffffffull) { set_error("cfg rescale: too many chunks"); return DPM_ERR_UNSUPPORTED; }
  auto al = [&](const void* q) { return (reinterpret_cast<uintptr_t>(q) & (dtype == DPM_F32 ? 31 : 15)) == 0; };
  const bool vec = per_sample % kPacket == 0 && al(ec) && al(eu);
  typedef void (*RKernel)(const RParams);
  RKernel k = with_packet_pair(dtype, dtype, [&](auto pair) -> RKernel {
    using T = typename decltype(pair)::TS;
    if (gscale != nullptr) return vec ? k_cfg_ratio_partial<T, true, true> : k_cfg_ratio_partial<T, false, true>;
    return vec ? k_cfg_ratio_partial<T, true> : k_cfg_ratio_partial<T, false>;
  });
  k<<<(unsigned)(p.n_samples * p.chunks), kEThreads, 0, stream>>>(p);
  k_cfg_ratio_final<<<(unsigned)((p.n_samples + kEThreads - 1) / kEThreads), kEThreads, 0, stream>>>(p);
  count_launch();
  count_launch();
  return DPM_OK;
}

}  // namespace dpm
