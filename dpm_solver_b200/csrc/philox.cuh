// philox.cuh -- torch.randn's normals, shared by the translation units that draw them (philox.cu, step_sde.cu).
//
// Host: ATen's launch geometry of a normal_ over a contiguous fp32 tensor (one segment per launch, split beyond
// 2^29 elements as TensorIterator splits it), defined in philox.cu.
// Device: the normals of that geometry formed from the Philox counter directly. Virtual thread idx of a launch with
// G = 256*grid threads draws, for its k-th curand_normal4, Philox4_32_10(counter = (offset/4 + k, idx), key = seed)
// -- what curand_init(seed, idx, offset) and k earlier calls leave in the state when offset % 4 == 0 -- and Box-Muller
// turns the block into 4 normals: lane ii is element idx + G*(4k + ii) of the segment.
#pragma once
#include <curand_kernel.h>
#include <stdint.h>

#include <vector>

namespace dpm {

constexpr int kPhiloxBlock = 256;   // ATen: block_size_bound
constexpr int kPhiloxUnroll = 4;    // curand_normal4 -> float4

struct NoiseSegment {
  uint64_t base, len;   // elements [base, base + len) of the noise tensor
  uint64_t offset;      // philox offset of this launch, relative to the generator's offset before the draw
  uint32_t grid;
};

// ATen's calc_execution_policy for one launch over `numel` elements on the current device
void launch_policy(uint64_t numel, uint32_t* grid, uint64_t* counter_offset);
// The launches ATen's distribution_nullary_kernel makes for a contiguous fp32 noise tensor of `numel` elements
// (appended to *segs when it is not NULL) and the total amount they advance the generator's philox offset by
uint64_t noise_segments(uint64_t numel, std::vector<NoiseSegment>* segs);

// Philox4_32_10 block `k` of virtual thread `idx` (offset4 = offset / 4)
__device__ __forceinline__ uint4 philox_block(uint64_t seed, uint64_t offset4, uint64_t idx, uint64_t k) {
  const uint64_t c = offset4 + k;
  const uint4 ctr = make_uint4((uint32_t)c, (uint32_t)(c >> 32), (uint32_t)idx, (uint32_t)(idx >> 32));
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  return curand_Philox4x32_10(ctr, key);
}

// curand's _curand_box_muller as nvcc compiles it with its default fma contraction, restated for a translation unit
// built with -fmad=false: the two sites that contraction fuses, the uniform u and the angle v, are spelled as fmas.
// (u's product is exact, v's is not: v is where an unfused product would move the normals.) logf, sqrtf and
// __sincosf compile to the same instructions either way.
__device__ __forceinline__ float2 box_muller(uint32_t x, uint32_t y) {
  const float u = __fmaf_rn((float)x, CURAND_2POW32_INV, CURAND_2POW32_INV / 2.0f);
  const float v = __fmaf_rn((float)y, CURAND_2POW32_INV_2PI, CURAND_2POW32_INV_2PI / 2.0f);
  const float s = sqrtf(-2.0f * logf(u));
  float sn, cs;
  __sincosf(v, &sn, &cs);
  return make_float2(sn * s, cs * s);
}

// curand_normal4 of the block, as torch's normal_ returns it: rand*1 + 0 under contraction, which maps -0 to +0
__device__ __forceinline__ void normal4(uint4 r, float (&z)[4]) {
  const float2 a = box_muller(r.x, r.y), b = box_muller(r.z, r.w);
  z[0] = __fadd_rn(a.x, 0.f);
  z[1] = __fadd_rn(a.y, 0.f);
  z[2] = __fadd_rn(b.x, 0.f);
  z[3] = __fadd_rn(b.y, 0.f);
}

}  // namespace dpm
