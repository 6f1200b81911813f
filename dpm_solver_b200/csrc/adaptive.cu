// adaptive.cu -- error estimate of the adaptive step-size solver (dpm_solver_adaptive,
// dpm_solver_pytorch.py:999-1001):
//   delta = max(atol, rtol * max(|x_lower|, |x_prev|))
//   E     = max_b sqrt( mean_b( ((x_higher - x_lower) / delta)^2 ) )
// The reference spends 9 full-tensor eager ops on it; here one streaming pass produces per-chunk
// partial sums (fixed chunking and a fixed reduction tree: deterministic, unlike atomics) and a
// one-CTA epilogue folds them per sample in index order, takes sqrt(mean) and the batch maximum.
// Algorithmic bytes: 3*s per element read, one float written.
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

}  // namespace dpm
