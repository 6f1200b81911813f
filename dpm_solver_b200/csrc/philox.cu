// philox.cu -- add_noise and the DiffEdit corrector with the Gaussian noise drawn INSIDE the kernel.
//
//   DPM_Solver.add_noise(x, t, noise=None)   dpm_solver_pytorch.py:1012-1030
//       noise = torch.randn((T, *x.shape), device=x.device);  xt[i] = alpha_t[i]*x + sigma_t[i]*noise[i]
//   DiffEdit corrector (examples/stable-diffusion/scripts/diffedit_inpaint.ipynb, `corrector_fn`;
//   sampler.stochastic_encode sampler.py:92-96):
//       x = x*mask + (1 - mask)*(alpha_t*x0 + sigma_t*randn_like(x0))
//
// The reference materialises the noise tensor (one full write + one full read) and runs 3 / 6 eager ops. Here
// each element's normal is produced in registers by the SAME generator torch.randn uses on CUDA -- curand's
// Philox4_32_10 through curand_normal4 (Box-Muller), with ATen's launch geometry replayed as a VIRTUAL
// geometry (ATen/native/cuda/DistributionTemplates.h: distribution_elementwise_grid_stride_kernel, block 256,
// grid = min(#SM * maxThreadsPerSM/256, ceil(numel/256)), unroll 4): virtual thread idx, iteration k, lane ii own
// element li = idx + G*(4k + ii), G = 256*grid, and read  curand_init(seed, idx, offset) -> k-th curand_normal4.
// So for a given (seed, offset) of the torch generator the result is bit-identical to
// torch.randn + the reference's op chain, and the caller advances the generator by the same counter offset
// ATen would have (dpm_philox_policy), keeping later torch RNG calls in sync.
//
// Above 2^29 elements the fp32 noise tensor no longer fits 32-bit byte offsets, and ATen's distribution_nullary_kernel
// splits it (TensorIterator::with_32bit_indexing): it advances the generator once by the whole tensor's counter
// offset, then halves the tensor depth first, left piece first, until every piece fits, and draws each piece as its
// own launch with its own grid and a fresh philox state taken from the generator. noise_segments() lists those
// pieces; launch_noise_philox replays each as one launch over [base, base + len) of the noise tensor.
#include <curand_kernel.h>

#include <vector>

#include "common.cuh"
#include "launch.cuh"
#include "philox.cuh"

namespace dpm {

constexpr int kMaxTimes = 16;

struct NoiseParams {
  const void* x;        // x (add_noise) / x0 (corrector), state dtype, n elements
  const void* xt;       // corrector: the current sample, state dtype, n elements; NULL = add_noise
  const float* mask;    // corrector: fp32 mask, mask_n elements, broadcast over the leading dims (element e -> e % mask_n)
  void* out;            // [T, n] (add_noise) or [n] (corrector), out dtype
  uint64_t n;           // elements of x
  uint64_t base;        // first element of the [T, n] noise tensor this launch draws
  uint64_t numel;       // elements this launch draws: [base, base + numel), all of T * n unless ATen splits it
  uint64_t mask_n;
  uint64_t seed, offset;
  int32_t x_dtype, out_dtype, t_count;
  float alpha[kMaxTimes], sigma[kMaxTimes];
};

__global__ void __launch_bounds__(kPhiloxBlock, 4) k_noise_philox(const __grid_constant__ NoiseParams p) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  curandStatePhilox4_32_10_t state;
  curand_init(p.seed, idx, p.offset, &state);
  const int64_t G = (int64_t)blockDim.x * gridDim.x;
  const int64_t numel = (int64_t)p.numel;
  const int64_t rounded = ((numel - 1) / (G * kPhiloxUnroll) + 1) * G * kPhiloxUnroll;
  for (int64_t linear = idx; linear < rounded; linear += G * kPhiloxUnroll) {
    const float4 r = curand_normal4(&state);
    const float rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int ii = 0; ii < kPhiloxUnroll; ++ii) {
      const int64_t li = linear + G * ii;
      if (li < numel) {
        const uint64_t g = p.base + (uint64_t)li;
        const uint64_t ti = g / p.n, e = g - ti * p.n;
        const float x = load_any(p.x, p.x_dtype, e);
        // alpha_t * x + sigma_t * noise (:1026), each product and the sum rounded separately. This file is
        // compiled WITH fma contraction (curand's Box-Muller must round like the one inside torch), so the
        // reference's unfused op chain is spelled with the never-contracted intrinsics.
        float v = __fadd_rn(__fmul_rn(p.alpha[ti], x), __fmul_rn(p.sigma[ti], rr[ii]));
        if (p.xt != nullptr) {
          const float m = p.mask[e % p.mask_n];
          const float xt = load_any(p.xt, p.x_dtype, e);
          v = __fadd_rn(__fmul_rn(xt, m), __fmul_rn(__fsub_rn(1.f, m), v));   // x * mask + (1 - mask) * stochastic_intermediate
        }
        store_any(p.out, p.out_dtype, (size_t)g, v);
      }
    }
  }
}

// ATen's calc_execution_policy for one launch over `numel` elements on the current device
void launch_policy(uint64_t numel, uint32_t* grid, uint64_t* counter_offset) {
  int dev = 0, max_thr = 2048;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&max_thr, cudaDevAttrMaxThreadsPerMultiProcessor, dev);
  const uint64_t by_size = (numel + kPhiloxBlock - 1) / kPhiloxBlock;
  const uint64_t by_dev = (uint64_t)sm_count() * (uint64_t)(max_thr / kPhiloxBlock);
  const uint32_t g = (uint32_t)(by_size < by_dev ? by_size : by_dev);
  *grid = g;
  *counter_offset = numel == 0 ? 0 : ((numel - 1) / ((uint64_t)kPhiloxBlock * g * kPhiloxUnroll) + 1) * 4;
}

// TensorIterator::can_use_32bit_indexing() of a contiguous fp32 tensor of len >= 1 elements
static bool fits_32bit_indexing(uint64_t len) {
  return len <= (uint64_t)INT32_MAX && 1 + (len - 1) * sizeof(float) <= (uint64_t)INT32_MAX;
}

// SplitUntil32Bit on the coalesced 1-D iterator: TensorIteratorBase::split gives the first len/2 elements to the
// piece it returns, which is drawn (and split further) before the rest. Each piece takes its counter offset from
// the generator in that order, after the whole tensor's.
static void split_segments(uint64_t base, uint64_t len, uint64_t* offset, std::vector<NoiseSegment>* segs) {
  if (!fits_32bit_indexing(len)) {
    split_segments(base, len / 2, offset, segs);
    split_segments(base + len / 2, len - len / 2, offset, segs);
    return;
  }
  NoiseSegment s = {base, len, *offset, 0};
  uint64_t co = 0;
  launch_policy(len, &s.grid, &co);
  *offset += co;
  if (segs != nullptr) segs->push_back(s);
}

// The launches ATen's distribution_nullary_kernel makes for a contiguous fp32 noise tensor of `numel` elements
// (appended to *segs when it is not NULL) and the total amount they advance the generator's philox offset by
uint64_t noise_segments(uint64_t numel, std::vector<NoiseSegment>* segs) {
  if (numel == 0) return 0;
  uint32_t grid = 0;
  uint64_t offset = 0;
  launch_policy(numel, &grid, &offset);
  if (fits_32bit_indexing(numel)) {
    if (segs != nullptr) segs->push_back({0, numel, 0, grid});
    return offset;
  }
  split_segments(0, numel, &offset, segs);
  return offset;
}

void philox_policy(uint64_t numel, uint32_t* grid, uint64_t* counter_offset) {
  uint64_t unsplit = 0;
  launch_policy(numel, grid, &unsplit);
  *counter_offset = noise_segments(numel, nullptr);
}

int launch_noise_philox(void* out, const void* x, const void* xt, const float* mask, uint64_t mask_n, uint64_t n,
                        int t_count, const float* alpha, const float* sigma, uint64_t seed, uint64_t offset,
                        int x_dtype, int out_dtype, cudaStream_t stream) {
  if (n == 0 || t_count == 0) return DPM_OK;
  if (t_count < 0 || t_count > kMaxTimes) { set_error("add_noise: between 1 and %d time labels per call", kMaxTimes); return DPM_ERR_UNSUPPORTED; }
  if (xt != nullptr && (t_count != 1 || mask == nullptr || mask_n == 0)) { set_error("corrector: one time label and a mask"); return DPM_ERR_ARG; }
  if (offset % 4 != 0) { set_error("philox offset must be a multiple of 4"); return DPM_ERR_ARG; }
  NoiseParams p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.xt = xt; p.mask = mask; p.out = out; p.n = n; p.numel = n * (uint64_t)t_count; p.mask_n = mask_n ? mask_n : 1;
  p.seed = seed; p.offset = offset; p.x_dtype = x_dtype; p.out_dtype = out_dtype; p.t_count = t_count;
  for (int i = 0; i < t_count; ++i) { p.alpha[i] = alpha[i]; p.sigma[i] = sigma[i]; }
  std::vector<NoiseSegment> segs;
  noise_segments(p.numel, &segs);
  for (const NoiseSegment& s : segs) {
    p.base = s.base;
    p.numel = s.len;
    p.offset = offset + s.offset;
    k_noise_philox<<<s.grid, kPhiloxBlock, 0, stream>>>(p);
    count_launch();
  }
  return DPM_OK;
}

}  // namespace dpm
