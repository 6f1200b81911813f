// step_sde.cu -- SDE-DPM-Solver++ (Lu et al. 2022, arXiv:2211.01095): the multistep update with its Gaussian noise
// drawn inside the launch (dpm_step_sde).
//
// Per element, in fp32 with every op rounded:   out = <the LIN1 / DIFF2 / MS3 expression of dpm_step> + cz*z
// where z is torch.randn's normal for the element (philox.cuh). The model stage is dpm_step's (fast_model8 /
// model_value / guided_value of common.cuh, unchanged), so the launch reads and writes exactly what the ODE launch
// does: x, the network outputs (or m0), the older buffers; out, out2, m_out. No noise byte touches memory.
//
// Mapping. ATen draws element li of a noise segment from virtual thread idx = li % G (G = 256*grid, a multiple of 256)
// as lane ii = j % 4 of its k-th curand_normal4, j = li / G, k = j / 4. One CUDA thread here owns the 8 consecutive
// virtual threads v0 .. v0+7 (v0 % 8 == 0) and one k: 8 Philox blocks give the 32 normals of the four 8-element
// packets that start at v0 + G*(4k + ii), ii = 0..3 -- one Philox block per 4 elements, as in torch, and the
// 128/256-bit packet accesses of the step kernels stay. A packet that crosses the end of the segment, a segment whose
// base is not a multiple of 8 (the halves ATen splits a tensor beyond 2^29 elements into), unaligned views and
// per-sample words over samples that do not hold whole packets take the element path (load_any / model_value).
#include "common.cuh"
#include "launch.cuh"
#include "philox.cuh"

namespace dpm {

constexpr int kSdeThreads = 256;

// the guidance kinds of the model stage (all NE == 2): the scalar combine, the rescaled one (dpm_step_rescaled), and
// per-sample words (dpm_step_guided / dpm_step_cfgzero / dpm_step_tcfg)
enum { kSdePlain = 0, kSdeRescale = 1, kSdeGuided = 2 };

struct SdeParams {
  KParams k;
  const float* z;       // materialised noise, fp32 [n] in storage order, or NULL: drawn here
  float cz;
  uint64_t seed, offset4;   // Philox key and offset / 4 of this segment
  uint64_t base, len;       // the segment: elements [base, base + len)
  uint64_t G;               // ATen's 256*grid for the segment
  uint64_t iters;           // ceil(len / (4G))
  int32_t vec;              // the packet path may serve whole packets of this segment
};

// the model stage and update of one element (the generic kernel's arithmetic, k_step_scalar)
__device__ __noinline__ void sde_element(const SdeParams& q, uint64_t i, float z) {
  const KParams& p = q.k;
  const int sd = p.state_dtype, md = p.model_dtype;
  const FormReads reads = form_reads(p.form);
  const float x = load_any(p.x, sd, i);
  const float m1 = reads.m1 ? load_any(p.m1, sd, i) : 0.f;
  const float m2 = reads.m2 ? load_any(p.m2, sd, i) : 0.f;
  float T0;
  if (p.n_model > 0) {
    const float xe = p.use_xe ? (p.xe_is_x ? x : load_any(p.xe, sd, i)) : 0.f;
    const float ec = load_any(p.ec, md, i);
    const float eu = p.n_model == 2 ? load_any(p.eu, md, i) : 0.f;
    const bool clamp = p.thr != nullptr;
    const uint64_t b = i / p.per_sample;
    const float thr = clamp ? p.thr[b] : 1.f;
    float mv;
    if (p.gscale != nullptr || p.zs != nullptr || p.td != nullptr) {
      const float r = p.zs != nullptr ? p.zs[b] : (p.td != nullptr ? p.td[2 * b] : (p.ratio != nullptr ? p.ratio[b] : 1.f));
      mv = model_value<2, false, false, kPgAny>(p, xe, ec, eu, thr, clamp, r,
                                                p.gscale != nullptr ? p.gscale[b] : p.guidance,
                                                p.td != nullptr ? p.td[2 * b + 1] : 0.f);
    } else if (p.ratio != nullptr) {
      mv = model_value<2, false, true>(p, xe, ec, eu, thr, clamp, p.ratio[b]);
    } else {
      mv = p.n_model == 2 ? model_value<2>(p, xe, ec, eu, thr, clamp) : model_value<1>(p, xe, ec, eu, thr, clamp);
    }
    T0 = round_any(sd, mv);
    if (p.m_out) store_any(p.m_out, sd, i, mv);
  } else {
    T0 = load_any(p.m0, sd, i);
  }
  float o;
  switch (p.form) {
    case DPM_FORM_LIN1: o = update_value<DPM_FORM_LIN1>(p, x, T0, m1, m2); break;
    case DPM_FORM_DIFF2: o = update_value<DPM_FORM_DIFF2>(p, x, T0, m1, m2); break;
    default: o = update_value<DPM_FORM_MS3>(p, x, T0, m1, m2); break;
  }
  o = o + q.cz * z;
  store_any(p.out, sd, i, o);
  if (p.out2) store_any(p.out2, sd, i, o);
}

// one 8-element packet pk (every stream 16/32-byte aligned): step_direct's model stage and update, then + cz*z
template <typename TE, typename TS, int NE, int FORM, bool FAST, int GK>
__device__ __forceinline__ void sde_packet(const SdeParams& q, uint64_t pk, const float (&z)[8]) {
  const KParams& p = q.k;
  constexpr bool kM1 = form_reads(FORM).m1, kM2 = form_reads(FORM).m2;
  const size_t e = (size_t)pk * kPacket;
  const bool sep_xe = (NE > 0) && p.use_xe && !p.xe_is_x;
  const bool clamp = (NE > 0) && (p.thr != nullptr);
  Raw<TS> rx, rxe, rm0, rm1, rm2;
  Raw<TE> rec, reu;
  // ---- every load of the packet first ----
  ldg_pk(rx, static_cast<const TS*>(p.x) + e);
  if (NE > 0) {
    ldg_pk(rec, static_cast<const TE*>(p.ec) + e);
    if (NE == 2) ldg_pk(reu, static_cast<const TE*>(p.eu) + e);
    if (sep_xe) ldg_pk(rxe, static_cast<const TS*>(p.xe) + e);
  } else {
    ldg_pk(rm0, static_cast<const TS*>(p.m0) + e);
  }
  if (kM1) ldg_pk(rm1, static_cast<const TS*>(p.m1) + e);
  if (kM2) ldg_pk(rm2, static_cast<const TS*>(p.m2) + e);
  float fx[8], fT[8], fm1[8], fm2[8], fo[8];
  unpack(rx, fx);
  if (kM1) unpack(rm1, fm1);
  if (kM2) unpack(rm2, fm2);
  if constexpr (NE > 0) {
    float fxe[8], fec[8], feu[8];
    unpack(rec, fec);
    if (NE == 2) unpack(reu, feu);
    if (sep_xe) {
      unpack(rxe, fxe);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) fxe[i] = fx[i];
    }
    // samples hold whole packets whenever a per-sample word or threshold is read here (the host routes the rest to
    // the element path): one scalar each per packet
    const uint32_t b = p.pk_per_sample ? (uint32_t)(pk / p.pk_per_sample) : 0u;
    if constexpr (FAST) {
      const float s_thr = clamp ? __ldg(p.thr + b) : 1.f;
      if constexpr (GK == kSdeGuided) {
        const float r = p.ratio != nullptr ? __ldg(p.ratio + b) : 1.f;
        fast_model8<NE, false, true>(p, fxe, fec, feu, clamp, s_thr, fT, r, __ldg(p.gscale + b));
      } else if constexpr (GK == kSdeRescale) {
        fast_model8<NE, true>(p, fxe, fec, feu, clamp, s_thr, fT, __ldg(p.ratio + b));
      } else {
        fast_model8<NE>(p, fxe, fec, feu, clamp, s_thr, fT);
      }
    } else if constexpr (GK == kSdeGuided) {
      const float gpk = p.gscale != nullptr ? __ldg(p.gscale + b) : p.guidance;
      const float rpk = p.zs != nullptr ? __ldg(p.zs + b) : (p.ratio != nullptr ? __ldg(p.ratio + b) : 1.f);
      const float tpk = clamp ? __ldg(p.thr + b) : 1.f;
      auto guided8 = [&](auto kind, float r, float r2) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          fT[i] = model_value<NE, false, false, decltype(kind)::value>(p, fxe[i], fec[i], feu[i], tpk, clamp, r, gpk,
                                                                       r2);
      };
      const int kind = pg_kind(p, gpk);
      if (kind == kPgBypass) guided8(std::integral_constant<int, kPgBypass>{}, rpk, 0.f);
      else if (kind == kPgRescale) guided8(std::integral_constant<int, kPgRescale>{}, rpk, 0.f);
      else if (kind == kPgZeroStar) guided8(std::integral_constant<int, kPgZeroStar>{}, rpk, 0.f);
      else if (kind == kPgTangential)
        guided8(std::integral_constant<int, kPgTangential>{}, __ldg(p.td + 2 * b), __ldg(p.td + 2 * b + 1));
      else guided8(std::integral_constant<int, kPgCombine>{}, rpk, 0.f);
    } else {
      // thresholds per packet when samples hold whole packets, else per element
      float thr8[8];
#pragma unroll
      for (int i = 0; i < 8; ++i)
        thr8[i] = !clamp ? 1.f : (p.pk_per_sample ? __ldg(p.thr + b) : __ldg(p.thr + (e + i) / p.per_sample));
      const float r = GK == kSdeRescale ? __ldg(p.ratio + b) : 1.f;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        fT[i] = model_value<NE, false, GK == kSdeRescale>(p, fxe[i], fec[i], NE == 2 ? feu[i] : 0.f, thr8[i], clamp, r);
    }
    Raw<TS> rmo;
    round_pack(rmo, fT);
    if (p.m_out != nullptr) stg_pk(static_cast<TS*>(p.m_out) + e, rmo);
  } else {
    unpack(rm0, fT);
  }
  if (FAST) {
    fast_update8<FORM>(p, fx, fT, fm1, fm2, fo);
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) fo[i] = update_value<FORM>(p, fx[i], fT[i], kM1 ? fm1[i] : 0.f, kM2 ? fm2[i] : 0.f);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) fo[i] = fo[i] + q.cz * z[i];
  Raw<TS> ro;
  pack(ro, fo);
  stg_pk(static_cast<TS*>(p.out) + e, ro);
  if (p.out2 != nullptr) stg_pk(static_cast<TS*>(p.out2) + e, ro);
}

template <typename TE, typename TS, int NE, int FORM, bool FAST, int GK>
__global__ void __launch_bounds__(kSdeThreads) k_step_sde(const __grid_constant__ SdeParams q) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t groups = q.G / 8;
  pdl_trigger();
  pdl_wait();
  if (t >= groups * q.iters) return;
  const uint64_t v0 = (t % groups) * 8, k = t / groups;
  float z[4][8];
  if (q.z == nullptr) {
#pragma unroll
    for (int v = 0; v < 8; ++v) {
      float w[4];
      normal4(philox_block(q.seed, q.offset4, v0 + v, k), w);
#pragma unroll
      for (int ii = 0; ii < 4; ++ii) z[ii][v] = w[ii];
    }
  }
#pragma unroll
  for (int ii = 0; ii < 4; ++ii) {
    const uint64_t li0 = v0 + q.G * (4 * k + ii);
    if (li0 >= q.len) break;
    const uint64_t e0 = q.base + li0;
    const bool whole = q.vec && li0 + 8 <= q.len;
    if (q.z != nullptr) {
      if (whole) {
        Raw<float> rz;
        ldg_pk(rz, q.z + e0);
        unpack(rz, z[ii]);
      } else {
#pragma unroll
        for (int v = 0; v < 8; ++v) z[ii][v] = li0 + v < q.len ? q.z[e0 + v] : 0.f;
      }
    }
    if (whole) {
      sde_packet<TE, TS, NE, FORM, FAST, GK>(q, e0 / kPacket, z[ii]);
    } else {
#pragma unroll
      for (int v = 0; v < 8; ++v)
        if (li0 + v < q.len) sde_element(q, e0 + v, z[ii][v]);
    }
  }
}

typedef void (*SdeKernel)(const SdeParams);

// the kernel of a launch: dtype pair, NE, form; FAST as dpm_step picks it (CFG-Zero* and TCFG words on the IEEE-division
// instantiations); other dtype pairs give the element-only instantiation
static SdeKernel pick_sde(const KParams& p) {
  const bool zt = p.zs != nullptr || p.td != nullptr;
  const bool guided = p.gscale != nullptr || zt, rs = p.ratio != nullptr && !guided;
  const bool fast = fast_path_ok(p) && !zt;
  return pick_step<SdeKernel>(p, [&](auto pair, auto ne, auto form) -> SdeKernel {
    using TE = typename decltype(pair)::TE;
    using TS = typename decltype(pair)::TS;
    constexpr int NE = decltype(ne)::value, FORM = decltype(form)::value;
    if constexpr (FORM != DPM_FORM_LIN1 && FORM != DPM_FORM_DIFF2 && FORM != DPM_FORM_MS3) {
      return nullptr;
    } else if constexpr (NE == 0) {
      return k_step_sde<TE, TS, 0, FORM, true, kSdePlain>;
    } else if constexpr (NE == 1) {
      return fast ? k_step_sde<TE, TS, 1, FORM, true, kSdePlain> : k_step_sde<TE, TS, 1, FORM, false, kSdePlain>;
    } else {
      if (guided)
        return fast ? k_step_sde<TE, TS, 2, FORM, true, kSdeGuided> : k_step_sde<TE, TS, 2, FORM, false, kSdeGuided>;
      if (rs)
        return fast ? k_step_sde<TE, TS, 2, FORM, true, kSdeRescale> : k_step_sde<TE, TS, 2, FORM, false, kSdeRescale>;
      return fast ? k_step_sde<TE, TS, 2, FORM, true, kSdePlain> : k_step_sde<TE, TS, 2, FORM, false, kSdePlain>;
    }
  });
}

int launch_step_sde(const KParams& p, const float* z, float cz, uint64_t seed, uint64_t offset, bool aligned_all,
                    cudaStream_t stream) {
  SdeParams q;
  memset(&q, 0, sizeof(q));
  q.k = p;
  q.z = z;
  q.cz = cz;
  q.seed = seed;
  SdeKernel k = pick_sde(p);
  const bool per_sample_words = p.thr != nullptr || p.ratio != nullptr || p.gscale != nullptr || p.zs != nullptr ||
                                p.td != nullptr;
  const bool vec = k != nullptr && aligned_all && !(per_sample_words && p.pk_per_sample == 0);
  if (k == nullptr) k = k_step_sde<float, float, 0, DPM_FORM_LIN1, true, kSdePlain>;   // other pairs: the element path
  std::vector<NoiseSegment> segs;
  if (z != nullptr) {   // a materialised draw: any geometry reads it; ATen's unsplit one
    NoiseSegment s = {0, p.n, 0, 0};
    uint64_t co = 0;
    launch_policy(p.n, &s.grid, &co);
    segs.push_back(s);
  } else {
    noise_segments(p.n, &segs);
  }
  for (const NoiseSegment& s : segs) {
    q.base = s.base;
    q.len = s.len;
    q.offset4 = (offset + s.offset) / 4;
    q.G = (uint64_t)kPhiloxBlock * s.grid;
    q.iters = (s.len + kPhiloxUnroll * q.G - 1) / (kPhiloxUnroll * q.G);
    q.vec = vec && s.base % kPacket == 0;
    const uint64_t threads = q.G / 8 * q.iters;
    const uint64_t grid = (threads + kSdeThreads - 1) / kSdeThreads;
    cudaError_t le = launch_pdl(k, (unsigned)grid, kSdeThreads, 0, stream, q);
    if (le != cudaSuccess) return launch_error("sde step launch failed", le);
    count_launch();
  }
  return 0;
}

}  // namespace dpm
