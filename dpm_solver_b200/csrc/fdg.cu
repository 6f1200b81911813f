// fdg.cu -- frequency-decoupled guidance (dpm_fdg_guided; Sadat, Vontobel, Salehi and Weber, "Guidance in the Frequency
// Domain Enables High-Fidelity Sampling at Low CFG Scales", 2025). Per plane (the last two dims of one sample and one
// channel), with d = c - u in fp32 and delta_l = fl32(w_l - w_{l-1}):
//   G_0 = d;  G_{l+1} = Down(G_l)                       l < N-1
//   E_{N-1} = delta_{N-1}*G_{N-1};  E_l = delta_l*G_l + Up(E_{l+1})     l = N-2 .. 1
//   g = (u + w_0*d) + Up(E_1)   (N >= 2),   g = u + w_0*d   (N == 1),   stored in the network's dtype
// Down and Up are the separable 6-tap / 4-tap polyphase filters of the header, horizontal pass first, reflect borders.
// One CTA per plane. c and u are read once, g written once (3*s_model bytes per element); every level lives in shared
// memory: region A holds d, then G_1 .. G_{N-1} (and E_l in place of G_l), then Up(E_1); region B holds the
// horizontal pass of each filter. Rows are padded to an odd stride, so that the filter passes (horizontal ones with
// lanes over rows, vertical ones with lanes over columns) are free of bank conflicts. Each thread owns NPK packets of 8
// consecutive plane elements and keeps u + w_0*d for them in registers between the load and the store; its stores of d
// and reads of Up(E_1) are 8 words apart from its neighbours', which costs bank conflicts in those two phases.
// Small CTAs (128 threads at 64 x 64) keep up to 6 planes in flight per SM; a persistent CTA prefetching the next
// plane with cp.async measured slower at 64 x 64 (DESIGN.md section 8 item 16).
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kFMaxLevels = DPM_FDG_MAX_LEVELS;
constexpr uint64_t kFMaxPlane = DPM_FDG_MAX_PLANE;

struct FParams {
  void* g;
  const void* ec;
  const void* eu;
  const float* scales;        // [n_samples][scale_stride] in device memory, or NULL: w
  uint64_t scale_stride;
  uint64_t planes_per_sample;
  int64_t sample_stride, plane_stride, h_stride, w_stride;   // elements
  float w[kFMaxLevels];       // shared scales (scales == NULL)
  int32_t H, W, levels;
  int32_t vec;                // planes dense row-major, plane bases 16-byte aligned, H*W % 8 == 0
};

__device__ __forceinline__ int refl(int j, int n) { return j < 0 ? -j : (j > n - 1 ? 2 * (n - 1) - j : j); }

// Down along one line of n (even) samples: outputs j0 .. j0+3 (those below n/2) from a[R(2*j0 - 2 + m)], m < 12.
// `at(k)` reads line sample k, `put(j, v)` writes output j.
template <typename At, typename Put>
__device__ __forceinline__ void down4(int j0, int n, At at, Put put) {
  const int nq = min(4, n / 2 - j0);
  const int lim = 2 * nq + 4;
  float a[12];
#pragma unroll
  for (int m = 0; m < 12; ++m) a[m] = m < lim ? at(refl(2 * j0 - 2 + m, n)) : 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (q < nq) {
      const float* t = a + 2 * q;
      float s = 0.03125f * t[0];
      s = s + 0.15625f * t[1];
      s = s + 0.3125f * t[2];
      s = s + 0.3125f * t[3];
      s = s + 0.15625f * t[4];
      s = s + 0.03125f * t[5];
      put(j0 + q, s);
    }
  }
}

// Up along one line of m (>= 3) samples: outputs 2*i0 .. 2*i0+3 (those below 2*m) from a[R(i0 - 2 + k)], k < 6.
template <typename At, typename Put>
__device__ __forceinline__ void up2(int i0, int m, At at, Put put) {
  const bool two = i0 + 1 < m;
  float a[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) a[k] = (k < 5 || two) ? at(refl(i0 - 2 + k, m)) : 0.f;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    if (q == 0 || two) {
      const float* t = a + q;
      float e = 0.015625f * t[0];
      e = e + 0.328125f * t[1];
      e = e + 0.546875f * t[2];
      e = e + 0.109375f * t[3];
      float o = 0.109375f * t[1];
      o = o + 0.546875f * t[2];
      o = o + 0.328125f * t[3];
      o = o + 0.015625f * t[4];
      put(2 * (i0 + q), e);
      put(2 * (i0 + q) + 1, o);
    }
  }
}

// src [h][w] (row stride ss) -> dst [h][w/2] (row stride ds): Down along rows; lanes over rows
__device__ void down_h(const float* src, int ss, float* dst, int ds, int h, int w) {
  const int nb = (w / 2 + 3) / 4;
  for (int idx = threadIdx.x; idx < h * nb; idx += blockDim.x) {
    const int r = idx % h, b = idx / h;
    const float* s = src + r * ss;
    float* d = dst + r * ds;
    down4(4 * b, w, [&](int k) { return s[k]; }, [&](int j, float v) { d[j] = v; });
  }
}

// src [h][w] -> dst [h/2][w]: Down along columns; lanes over columns
__device__ void down_v(const float* src, int ss, float* dst, int ds, int h, int w) {
  const int nb = (h / 2 + 3) / 4;
  for (int idx = threadIdx.x; idx < w * nb; idx += blockDim.x) {
    const int c = idx % w, b = idx / w;
    down4(4 * b, h, [&](int k) { return src[k * ss + c]; }, [&](int j, float v) { dst[j * ds + c] = v; });
  }
}

// src [h][w] -> dst [h][2w]: Up along rows; lanes over rows
__device__ void up_h(const float* src, int ss, float* dst, int ds, int h, int w) {
  const int nb = (w + 1) / 2;
  for (int idx = threadIdx.x; idx < h * nb; idx += blockDim.x) {
    const int r = idx % h, b = idx / h;
    const float* s = src + r * ss;
    float* d = dst + r * ds;
    up2(2 * b, w, [&](int k) { return s[k]; }, [&](int j, float v) { d[j] = v; });
  }
}

// src [h][w] -> dst [2h][w]: Up along columns; lanes over columns. combine: dst = delta*dst + Up (E_l in place of G_l)
__device__ void up_v(const float* src, int ss, float* dst, int ds, int h, int w, float delta, bool combine) {
  const int nb = (h + 1) / 2;
  for (int idx = threadIdx.x; idx < w * nb; idx += blockDim.x) {
    const int c = idx % w, b = idx / w;
    up2(2 * b, h, [&](int k) { return src[k * ss + c]; }, [&](int j, float v) {
      float* o = dst + j * ds + c;
      *o = combine ? delta * *o + v : v;
    });
  }
}

__host__ __device__ __forceinline__ int fdg_stride(int w) { return w + 1; }   // odd row stride of every level

// floats of dynamic shared memory: region A (H rows of W + 1) and region B (H rows of W/2 + 1, which also holds the
// H/2 rows of W + 1 of the last Up's horizontal pass)
static size_t fdg_smem_floats(int H, int W, int levels) {
  if (levels == 1) return 0;
  return (size_t)H * fdg_stride(W) + (size_t)H * fdg_stride(W / 2);
}

// THREADS x NPK x 8 >= H*W; MINB resident CTAs per SM (the register bound of __launch_bounds__)
template <typename TE, int NPK, int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) k_fdg_guided(const __grid_constant__ FParams p) {
  extern __shared__ float smem[];
  const int H = p.H, W = p.W, L = p.levels, HW = H * W;
  float* A = smem;
  float* Bs = smem + (size_t)H * fdg_stride(W);
  auto goff = [&](int64_t base, int e) -> int64_t {
    const int r = e / W, c = e - r * W;
    return base + (int64_t)r * p.h_stride + (int64_t)c * p.w_stride;
  };
  const uint64_t plane = blockIdx.x;
  // (the plane's base offset and scales are recomputed where used: held across the pyramid they would spill)
  auto sample = [&]() -> uint64_t { return plane / p.planes_per_sample; };
  auto plane_base = [&]() -> int64_t {
    return (int64_t)sample() * p.sample_stride + (int64_t)(plane % p.planes_per_sample) * p.plane_stride;
  };
  auto scale = [&](int l) -> float { return p.scales != nullptr ? p.scales[sample() * p.scale_stride + l] : p.w[l]; };

  // ---- load: d to region A, u + w_0*d in registers ----
  float keep[NPK][8];
  {
  const int64_t base = plane_base();
  const float w0 = scale(0);
#pragma unroll
  for (int k = 0; k < NPK; ++k) {
    const int e0 = (k * THREADS + threadIdx.x) * 8;
    if (e0 >= HW) continue;
    float fc[8], fu[8];
    if (p.vec) {
      Raw<TE> rc, ru;
      ldg_pk(rc, static_cast<const TE*>(p.ec) + base + e0);
      ldg_pk(ru, static_cast<const TE*>(p.eu) + base + e0);
      unpack(rc, fc);
      unpack(ru, fu);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        fc[i] = e0 + i < HW ? load_any(p.ec, Traits<TE>::kCode, goff(base, e0 + i)) : 0.f;
        fu[i] = e0 + i < HW ? load_any(p.eu, Traits<TE>::kCode, goff(base, e0 + i)) : 0.f;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = fc[i] - fu[i];
      keep[k][i] = fu[i] + w0 * d;
      if (L > 1 && e0 + i < HW) {
        const int r = (e0 + i) / W;
        A[r * fdg_stride(W) + (e0 + i - r * W)] = d;
      }
    }
  }
  }

  if (L > 1) {
    // ---- pyramid of d: G_l at A + off(l) (G_0 = d at offset 0, overwritten by G_1 .. once G_1's input is in B) ----
    auto off = [&](int l) {
      int o = 0;
      for (int k = 1; k < l; ++k) o += (H >> k) * fdg_stride(W >> k);
      return o;
    };
    __syncthreads();
    down_h(A, fdg_stride(W), Bs, fdg_stride(W / 2), H, W);
    __syncthreads();
    down_v(Bs, fdg_stride(W / 2), A + off(1), fdg_stride(W / 2), H, W / 2);
    __syncthreads();
    for (int l = 1; l + 1 < L; ++l) {
      const int h = H >> l, w = W >> l;
      down_h(A + off(l), fdg_stride(w), Bs, fdg_stride(w / 2), h, w);
      __syncthreads();
      down_v(Bs, fdg_stride(w / 2), A + off(l + 1), fdg_stride(w / 2), h, w / 2);
      __syncthreads();
    }
    // ---- E_{N-1} = delta_{N-1}*G_{N-1}, then E_l = delta_l*G_l + Up(E_{l+1}) in place of G_l ----
    {
      const int h = H >> (L - 1), w = W >> (L - 1);
      const float dl = scale(L - 1) - scale(L - 2);
      float* E = A + off(L - 1);
      for (int idx = threadIdx.x; idx < h * w; idx += blockDim.x) {
        const int r = idx / w, c = idx - r * w;
        E[r * fdg_stride(w) + c] = dl * E[r * fdg_stride(w) + c];
      }
      __syncthreads();
    }
    for (int l = L - 2; l >= 1; --l) {
      const int h = H >> (l + 1), w = W >> (l + 1);
      up_h(A + off(l + 1), fdg_stride(w), Bs, fdg_stride(2 * w), h, w);
      __syncthreads();
      up_v(Bs, fdg_stride(2 * w), A + off(l), fdg_stride(2 * w), h, 2 * w, scale(l) - scale(l - 1), true);
      __syncthreads();
    }
    // ---- Up(E_1) to region A (row stride W + 1) ----
    up_h(A + off(1), fdg_stride(W / 2), Bs, fdg_stride(W), H / 2, W / 2);
    __syncthreads();
    up_v(Bs, fdg_stride(W), A, fdg_stride(W), H / 2, W, 0.f, false);
    __syncthreads();
  }

  // ---- store g = keep + Up(E_1) in the network's dtype ----
  const int64_t base = plane_base();
#pragma unroll
  for (int k = 0; k < NPK; ++k) {
    const int e0 = (k * THREADS + threadIdx.x) * 8;
    if (e0 >= HW) continue;
    float g[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      g[i] = keep[k][i];
      if (L > 1 && e0 + i < HW) {
        const int r = (e0 + i) / W;
        g[i] = g[i] + A[r * fdg_stride(W) + (e0 + i - r * W)];
      }
    }
    if (p.vec) {
      Raw<TE> rg;
      pack(rg, g);
      stg_pk(static_cast<TE*>(p.g) + base + e0, rg);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (e0 + i < HW) store_any(p.g, Traits<TE>::kCode, goff(base, e0 + i), g[i]);
    }
  }
}

int fdg_supported(uint64_t H, uint64_t W, int levels, int model_dtype) {
  if (model_dtype != DPM_F32 && model_dtype != DPM_BF16 && model_dtype != DPM_F16) {
    set_error("fdg: bad model dtype %d", model_dtype);
    return DPM_ERR_ARG;
  }
  if (levels < 1 || levels > kFMaxLevels) {
    set_error("fdg: %d levels; 1 to %d are supported", levels, kFMaxLevels);
    return DPM_ERR_ARG;
  }
  const uint64_t f = 1ull << (levels - 1);
  if (H % f || W % f || H / f < 3 || W / f < 3) {
    set_error("fdg: a %llu x %llu plane with %d levels: H and W must be divisible by 2^(levels-1) = %llu, with a "
              "quotient of at least 3", (unsigned long long)H, (unsigned long long)W, levels, (unsigned long long)f);
    return DPM_ERR_ARG;
  }
  if (H > kFMaxPlane || W > kFMaxPlane || H * W > kFMaxPlane) {   // (bounded first: the product cannot wrap)
    set_error("fdg: a %llu x %llu plane exceeds %llu elements (H*W; 128 x 128 at most)", (unsigned long long)H,
              (unsigned long long)W, (unsigned long long)kFMaxPlane);
    return DPM_ERR_ARG;
  }
  return DPM_OK;
}

int launch_fdg_guided(void* g, const void* ec, const void* eu, int model_dtype, uint64_t planes, uint64_t H, uint64_t W,
                      int64_t sample_stride, int64_t plane_stride, int64_t h_stride, int64_t w_stride, int levels,
                      const float* scales, uint64_t scale_stride, uint64_t planes_per_sample, cudaStream_t stream) {
  if (const int rc = fdg_supported(H, W, levels, model_dtype)) return rc;
  if (planes == 0) return DPM_OK;
  if (!g || !ec || !eu || !scales) { set_error("fdg: NULL tensor or scales"); return DPM_ERR_ARG; }
  if (planes_per_sample == 0 || planes % planes_per_sample || (scale_stride != 0 && scale_stride < (uint64_t)levels)) {
    set_error("fdg: planes_per_sample must divide planes, and scale_stride be 0 or at least levels");
    return DPM_ERR_ARG;
  }
  if (planes > 0x7fffffffull) { set_error("fdg: more than 2^31 - 1 planes"); return DPM_ERR_UNSUPPORTED; }
  FParams p;
  memset(&p, 0, sizeof(p));
  p.g = g; p.ec = ec; p.eu = eu;
  p.planes_per_sample = planes_per_sample;
  p.sample_stride = sample_stride; p.plane_stride = plane_stride; p.h_stride = h_stride; p.w_stride = w_stride;
  p.H = (int32_t)H; p.W = (int32_t)W; p.levels = levels;
  if (scale_stride == 0) {
    for (int l = 0; l < levels; ++l) p.w[l] = scales[l];     // shared scales: host memory, by value
  } else {
    p.scales = scales; p.scale_stride = scale_stride;
  }
  const uintptr_t sz = model_dtype == DPM_F32 ? 4 : 2;
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vec = w_stride == 1 && h_stride == (int64_t)W && (H * W) % 8 == 0 && al(g) && al(ec) && al(eu) &&
          ((uint64_t)sample_stride * sz) % 16 == 0 && ((uint64_t)plane_stride * sz) % 16 == 0;
  typedef void (*FKernel)(const FParams);
  // CTA shapes: (NPK, THREADS, MINB) = (4, 128, 6) up to 64 x 64, (4, 256, 3) up to 8192 elements, (2, 1024, 1) up to
  // 128 x 128 (fewer threads with more packets each there spill; see DESIGN.md)
  const uint64_t packets = (H * W + 7) / 8;
  const int shape = packets <= 512 ? 0 : packets <= 1024 ? 1 : 2;
  const int threads = shape == 0 ? 128 : shape == 1 ? 256 : 1024;
  FKernel k = nullptr;
  auto pick = [&](auto te) -> FKernel {
    using TE = decltype(te);
    return shape == 0 ? k_fdg_guided<TE, 4, 128, 6> : shape == 1 ? k_fdg_guided<TE, 4, 256, 3>
                                                                  : k_fdg_guided<TE, 2, 1024, 1>;
  };
  if (model_dtype == DPM_F32) k = pick(float{});
  else if (model_dtype == DPM_BF16) k = pick(__nv_bfloat16{});
  else k = pick(__half{});
  const size_t smem = fdg_smem_floats((int)H, (int)W, levels) * sizeof(float);
  if (smem > 48 * 1024) {
    if (const int rc = ensure_max_smem(reinterpret_cast<const void*>(k))) return rc;
  }
  k<<<(unsigned)planes, threads, smem, stream>>>(p);
  count_launch();
  return DPM_OK;
}

}  // namespace dpm
