// step_multi.cu -- multi-condition classifier-free guidance fused into the step (dpm_step_multi), and the (K+1)-way
// copy of the first network input (dpm_replicate).
//
// The network runs once on cat([x]*(K+1)) with the conditions cat([uc, c1, ..., cK]) and returns K+1 blocks: eps_u
// first, then one per condition. Per element the kernel converts each block by the parameterisation (noise_pred_fn
// :288-298, as the reference converts the whole batch), forms
//   eps = eps_u;  eps = eps + s_k*(eps_k - eps_u),  k = 1..K          (every difference, product and sum rounded)
// -- torch's eager `eu + s1*(e1 - eu) + s2*(e2 - eu)` in fp32 -- then eps->x0 (:439), the thresholding clamp (:424) and
// the update, and writes m_out, x_t, and x_t again into the K replica blocks of the next network input (block 0 is x_t
// itself). Algorithmic traffic of an order-2 multistep step: x, K+1 outputs and m1 read, m_out, x_t and K replicas
// written: (2K + 5)*s bytes per element.
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kMultiUnroll = 2;
constexpr int kMultiThreads = 256;

// FAST: param == NOISE (the conversion is the identity) or FLOW / EDM (each block converted by flow8, one uniform branch per
// packet, no division), exact constant division, a clamp threshold uniform per packet (fast_path_ok). FAST = false:
// every parameterisation, per-element thresholds, IEEE division.
template <typename TE, typename TS, int FORM, bool FAST>
__global__ void __launch_bounds__(kMultiThreads) k_step_multi(const __grid_constant__ MultiParams mp) {
  const KParams& p = mp.k;
  constexpr bool kX = form_reads(FORM).x, kM1 = form_reads(FORM).m1, kM2 = form_reads(FORM).m2;
  const TS* __restrict__ gx = static_cast<const TS*>(p.x);
  const TS* __restrict__ gxe = static_cast<const TS*>(p.xe);
  const TS* __restrict__ gm1 = static_cast<const TS*>(p.m1);
  const TS* __restrict__ gm2 = static_cast<const TS*>(p.m2);
  const TE* __restrict__ geu = static_cast<const TE*>(p.eu);
  TS* __restrict__ gmo = static_cast<TS*>(p.m_out);
  TS* __restrict__ go = static_cast<TS*>(p.out);
  const int nc = mp.n_cond;

  const uint32_t npk = p.npk;
  const uint32_t tile_pk = blockDim.x * kMultiUnroll;
  const bool sep_xe = p.use_xe && !(kX && p.xe_is_x);
  const bool clamp = p.thr != nullptr;
  pdl_trigger();
  pdl_wait();

  for (uint64_t tile0 = (uint64_t)blockIdx.x * tile_pk; tile0 < npk; tile0 += (uint64_t)gridDim.x * tile_pk) {
    Raw<TS> rx[kMultiUnroll], rxe[kMultiUnroll], rm1[kMultiUnroll], rm2[kMultiUnroll];
    Raw<TE> reu[kMultiUnroll], rec[kMultiUnroll][kMaxCond];
    // ---- issue every load of the tile ----
#pragma unroll
    for (int u = 0; u < kMultiUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        if (kX) ldg_pk(rx[u], gx + e);
        ldg_pk(reu[u], geu + e);
#pragma unroll
        for (int k = 0; k < kMaxCond; ++k)
          if (k < nc) ldg_pk(rec[u][k], static_cast<const TE*>(mp.ec[k]) + e);
        if (sep_xe) ldg_pk(rxe[u], gxe + e);
        if (kM1) ldg_pk(rm1[u], gm1 + e);
        if (kM2) ldg_pk(rm2[u], gm2 + e);
      }
    }
    // ---- compute + store ----
#pragma unroll
    for (int u = 0; u < kMultiUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        float fx[8], fxe[8], fT[8], fm1[8], fm2[8], fo[8], fu[8], g[8];
        if (kX) unpack(rx[u], fx);
        if (kM1) unpack(rm1[u], fm1);
        if (kM2) unpack(rm2[u], fm2);
        if (sep_xe) {
          unpack(rxe[u], fxe);
        } else if (kX) {
#pragma unroll
          for (int i = 0; i < 8; ++i) fxe[i] = fx[i];
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) fxe[i] = 0.f;
        }
        unpack(reu[u], fu);
        if (FAST) {
          const bool flow = direct_param(p.param);
          if (flow) flow8(p, fxe, fu);
#pragma unroll
          for (int i = 0; i < 8; ++i) g[i] = fu[i];
#pragma unroll
          for (int k = 0; k < kMaxCond; ++k) {
            if (k < nc) {
              float fc[8];
              unpack(rec[u][k], fc);
              if (flow) flow8(p, fxe, fc);
              const float s = mp.s[k];
#pragma unroll
              for (int i = 0; i < 8; ++i) g[i] = g[i] + s * (fc[i] - fu[i]);
            }
          }
          const float s_thr = clamp ? __ldg(p.thr + (uint32_t)pk / p.pk_per_sample) : 1.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) fT[i] = g[i];
          fast_finish8(p, fxe, clamp, s_thr, fT);   // eps->x0 (a FLOW or EDM value is x0 already) and the clamp
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            fu[i] = convert_param(p, fu[i], fxe[i]);
            g[i] = fu[i];
          }
#pragma unroll
          for (int k = 0; k < kMaxCond; ++k) {
            if (k < nc) {
              float fc[8];
              unpack(rec[u][k], fc);
              const float s = mp.s[k];
#pragma unroll
              for (int i = 0; i < 8; ++i) g[i] = g[i] + s * (convert_param(p, fc[i], fxe[i]) - fu[i]);
            }
          }
          float thr8[8];
          if (clamp) {
            if (p.pk_per_sample != 0) {
              const float tpk = __ldg(p.thr + (uint32_t)(pk / p.pk_per_sample));
#pragma unroll
              for (int i = 0; i < 8; ++i) thr8[i] = tpk;
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i) thr8[i] = __ldg(p.thr + (e + i) / p.per_sample);
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) fT[i] = finish_x0(p, g[i], fxe[i], clamp ? thr8[i] : 1.f, clamp);
        }
        Raw<TS> rmo;
        round_pack(rmo, fT);
        if (gmo != nullptr) stg_pk(gmo + e, rmo);
        if (FORM != DPM_FORM_NONE) {
          if (FAST) {
            fast_update8<FORM>(p, fx, fT, fm1, fm2, fo);
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) fo[i] = update_value<FORM>(p, fx[i], fT[i], kM1 ? fm1[i] : 0.f, kM2 ? fm2[i] : 0.f);
          }
          Raw<TS> ro;
          pack(ro, fo);
          stg_pk(go + e, ro);
#pragma unroll
          for (int k = 0; k < kMaxCond; ++k)
            if (k < nc && mp.rep[k] != nullptr) stg_pk(static_cast<TS*>(mp.rep[k]) + e, ro);
        }
      }
    }
  }
}

// generic element-wise variant: any dtype pair, any alignment, tails, and dev_coef launches (scalars from the adaptive
// controller's coefficient block, common layout of k_step_scalar)
__global__ void __launch_bounds__(256) k_step_multi_scalar(const __grid_constant__ MultiParams mpc) {
  KParams p = mpc.k;
  if (p.dev_coef != nullptr) {
    const float* c = p.dev_coef;
    p.a = c[0]; p.c0 = c[1]; p.c1 = c[2]; p.c2 = c[3];
    p.w0 = c[4]; p.w1 = c[5]; p.w2 = c[6]; p.w3 = c[7]; p.w4 = c[8];
    p.alpha_e = c[9]; p.sigma_e = c[10];
    p.fast_div = 0;
  }
  const int sd = p.state_dtype, md = p.model_dtype, nc = mpc.n_cond;
  const FormReads reads = form_reads(p.form);
  const bool clamp = p.thr != nullptr;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (size_t)gridDim.x * blockDim.x) {
    const float x = reads.x ? load_any(p.x, sd, i) : 0.f;
    const float m1 = reads.m1 ? load_any(p.m1, sd, i) : 0.f;
    const float m2 = reads.m2 ? load_any(p.m2, sd, i) : 0.f;
    const float xe = p.use_xe ? ((reads.x && p.xe_is_x) ? x : load_any(p.xe, sd, i)) : 0.f;
    const float eu = convert_param(p, load_any(p.eu, md, i), xe);
    float eps = eu;
    for (int k = 0; k < nc; ++k)
      eps = eps + mpc.s[k] * (convert_param(p, load_any(mpc.ec[k], md, i), xe) - eu);
    const float mv = finish_x0(p, eps, xe, clamp ? p.thr[(i + p.elem_offset) / p.per_sample] : 1.f, clamp);
    if (p.m_out) store_any(p.m_out, sd, i, mv);
    const float T0 = round_any(sd, mv);
    float o;
    switch (p.form) {
      case DPM_FORM_LIN1: o = update_value<DPM_FORM_LIN1>(p, x, T0, m1, m2); break;
      case DPM_FORM_LIN2: o = update_value<DPM_FORM_LIN2>(p, x, T0, m1, m2); break;
      case DPM_FORM_LIN3: o = update_value<DPM_FORM_LIN3>(p, x, T0, m1, m2); break;
      case DPM_FORM_DIFF2: o = update_value<DPM_FORM_DIFF2>(p, x, T0, m1, m2); break;
      case DPM_FORM_MS3: o = update_value<DPM_FORM_MS3>(p, x, T0, m1, m2); break;
      case DPM_FORM_SS3T: o = update_value<DPM_FORM_SS3T>(p, x, T0, m1, m2); break;
      default: continue;
    }
    store_any(p.out, sd, i, o);
    for (int k = 0; k < nc; ++k)
      if (mpc.rep[k] != nullptr) store_any(mpc.rep[k], sd, i, o);
  }
}

typedef void (*MultiKernel)(const MultiParams);

int launch_step_multi(const MultiParams& mp, const Tuning& t, cudaStream_t stream) {
  const KParams& p = mp.k;
  const bool fast = fast_path_ok(p);
  MultiKernel k = with_packet_pair(p.model_dtype, p.state_dtype, [&](auto pair) -> MultiKernel {
    using TE = typename decltype(pair)::TE;
    using TS = typename decltype(pair)::TS;
    return with_form(p.form, [&](auto form) -> MultiKernel {
      constexpr int FORM = decltype(form)::value;
      return fast ? k_step_multi<TE, TS, FORM, true> : k_step_multi<TE, TS, FORM, false>;
    });
  });
  if (k == nullptr) return 1;  // other dtype pairs: the generic kernel
  const int threads = t.threads > 0 && t.threads <= kMultiThreads ? t.threads : kMultiThreads;
  const uint64_t tile_pk = (uint64_t)threads * kMultiUnroll;
  const uint64_t tiles = ((uint64_t)p.npk + tile_pk - 1) / tile_pk;
  const uint64_t cap = t.ctas_per_sm > 0 ? (uint64_t)sm_count() * t.ctas_per_sm : tiles;
  const uint32_t grid = (uint32_t)(tiles < cap ? tiles : cap);
  if (grid == 0) return 0;
  cudaError_t le = launch_pdl(k, grid, (unsigned)threads, 0, stream, mp);
  if (le != cudaSuccess) return launch_error("multi-condition step launch failed", le);
  count_launch();
  return 0;
}

int launch_step_multi_scalar(const MultiParams& mp, cudaStream_t stream) {
  if (mp.k.n == 0) return 0;
  const int threads = 256;
  const uint64_t blocks = (mp.k.n + threads - 1) / threads;
  const uint64_t cap = (uint64_t)sm_count() * 8;
  const uint32_t grid = (uint32_t)(blocks < cap ? blocks : cap);
  k_step_multi_scalar<<<grid, threads, 0, stream>>>(mp);
  count_launch();
  return 0;
}

// ---- dpm_step_multi_masked: the combine above with s_k*m_k(i) in place of s_k ----------------------------------------
// Per element, in fp32 with each op rounded: w = s_k*m_k(i); eps = eps + w*(eps_k - eps_u). A map of ones gives w == s_k
// exactly, so the result is k_step_multi's. Algorithmic traffic: k_step_multi's plus the weights (one word per sample and
// condition for period 1; a shared map is read once per launch and then served by L2).

// g += s_k*m_k(i)*(c - u) over the packet at packet rpk of sample b (samples hold whole packets), c and u converted.
// Without a map the weight is s_k itself; period 1: one weight for the packet; period % 8 == 0: two aligned 16-byte
// loads, each applied to its half of the packet as it arrives.
__device__ __forceinline__ void combine_packet(const MaskedParams& q, int k, uint32_t b, uint32_t rpk, float g[8],
                                               const float fc[8], const float fu[8]) {
  const float s = q.m.s[k];
  const float* w = q.w[k];
  if (w == nullptr || q.period[k] == 1) {
    const float wv = w == nullptr ? s : s * __ldg(w + (uint64_t)b * q.sstride[k]);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = g[i] + wv * (fc[i] - fu[i]);
  } else {
    const uint32_t ppk = (uint32_t)(q.period[k] / kPacket);
    const float4* w4 = reinterpret_cast<const float4*>(w + (uint64_t)b * q.sstride[k] + (uint64_t)(rpk % ppk) * kPacket);
    const float4 lo = __ldg(w4);
    g[0] = g[0] + (s * lo.x) * (fc[0] - fu[0]);
    g[1] = g[1] + (s * lo.y) * (fc[1] - fu[1]);
    g[2] = g[2] + (s * lo.z) * (fc[2] - fu[2]);
    g[3] = g[3] + (s * lo.w) * (fc[3] - fu[3]);
    const float4 hi = __ldg(w4 + 1);
    g[4] = g[4] + (s * hi.x) * (fc[4] - fu[4]);
    g[5] = g[5] + (s * hi.y) * (fc[5] - fu[5]);
    g[6] = g[6] + (s * hi.z) * (fc[6] - fu[6]);
    g[7] = g[7] + (s * hi.w) * (fc[7] - fu[7]);
  }
}

// the weight of condition k at global element gi, any period (the generic kernel)
__device__ __forceinline__ float elem_weight(const MaskedParams& q, int k, uint64_t gi) {
  const float s = q.m.s[k];
  const float* w = q.w[k];
  if (w == nullptr) return s;
  const uint64_t ps = q.m.k.per_sample;
  const uint64_t b = gi / ps;
  return s * w[b * q.sstride[k] + (gi - b * ps) % q.period[k]];
}

// FAST as k_step_multi. The weights are loaded in the compute phase: a shared map is an L2 hit, and holding both
// packets' weights in flight next to K + 1 outputs would cost registers at K = 4.
template <typename TE, typename TS, int FORM, bool FAST>
__global__ void __launch_bounds__(kMultiThreads) k_step_multi_masked(const __grid_constant__ MaskedParams q) {
  const MultiParams& mp = q.m;
  const KParams& p = mp.k;
  constexpr bool kX = form_reads(FORM).x, kM1 = form_reads(FORM).m1, kM2 = form_reads(FORM).m2;
  const TS* __restrict__ gx = static_cast<const TS*>(p.x);
  const TS* __restrict__ gxe = static_cast<const TS*>(p.xe);
  const TS* __restrict__ gm1 = static_cast<const TS*>(p.m1);
  const TS* __restrict__ gm2 = static_cast<const TS*>(p.m2);
  const TE* __restrict__ geu = static_cast<const TE*>(p.eu);
  TS* __restrict__ gmo = static_cast<TS*>(p.m_out);
  TS* __restrict__ go = static_cast<TS*>(p.out);
  const int nc = mp.n_cond;

  const uint32_t npk = p.npk;
  const uint32_t tile_pk = blockDim.x * kMultiUnroll;
  const bool sep_xe = p.use_xe && !(kX && p.xe_is_x);
  const bool clamp = p.thr != nullptr;
  pdl_trigger();
  pdl_wait();

  for (uint64_t tile0 = (uint64_t)blockIdx.x * tile_pk; tile0 < npk; tile0 += (uint64_t)gridDim.x * tile_pk) {
    Raw<TS> rx[kMultiUnroll], rxe[kMultiUnroll], rm1[kMultiUnroll], rm2[kMultiUnroll];
    Raw<TE> reu[kMultiUnroll], rec[kMultiUnroll][kMaxCond];
    // ---- issue every load of the tile ----
#pragma unroll
    for (int u = 0; u < kMultiUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        if (kX) ldg_pk(rx[u], gx + e);
        ldg_pk(reu[u], geu + e);
#pragma unroll
        for (int k = 0; k < kMaxCond; ++k)
          if (k < nc) ldg_pk(rec[u][k], static_cast<const TE*>(mp.ec[k]) + e);
        if (sep_xe) ldg_pk(rxe[u], gxe + e);
        if (kM1) ldg_pk(rm1[u], gm1 + e);
        if (kM2) ldg_pk(rm2[u], gm2 + e);
      }
    }
    // ---- compute + store ----
#pragma unroll
    for (int u = 0; u < kMultiUnroll; ++u) {
      const uint64_t pk64 = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk64 < npk) {
        const uint32_t pk = (uint32_t)pk64;   // (< npk: 32 bits, one register less at the K = 4 peak)
        const size_t e = (size_t)pk * kPacket;
        // (pk_per_sample is 0 only when no condition has a map)
        const uint32_t b = p.pk_per_sample != 0 ? pk / p.pk_per_sample : 0u;
        float fx[8], fxe[8], fT[8], fm1[8], fm2[8], fo[8], fu[8], g[8];
        if (kX) unpack(rx[u], fx);
        if (kM1) unpack(rm1[u], fm1);
        if (kM2) unpack(rm2[u], fm2);
        if (sep_xe) {
          unpack(rxe[u], fxe);
        } else if (kX) {
#pragma unroll
          for (int i = 0; i < 8; ++i) fxe[i] = fx[i];
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) fxe[i] = 0.f;
        }
        unpack(reu[u], fu);
        if (FAST) {
          const bool flow = direct_param(p.param);
          if (flow) flow8(p, fxe, fu);
#pragma unroll
          for (int i = 0; i < 8; ++i) g[i] = fu[i];
#pragma unroll
          for (int k = 0; k < kMaxCond; ++k) {
            if (k < nc) {
              float fc[8];
              unpack(rec[u][k], fc);
              if (flow) flow8(p, fxe, fc);
              combine_packet(q, k, b, pk - b * p.pk_per_sample, g, fc, fu);
            }
          }
          const float s_thr = clamp ? __ldg(p.thr + b) : 1.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) fT[i] = g[i];
          fast_finish8(p, fxe, clamp, s_thr, fT);   // eps->x0 (a FLOW or EDM value is x0 already) and the clamp
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            fu[i] = convert_param(p, fu[i], fxe[i]);
            g[i] = fu[i];
          }
#pragma unroll
          for (int k = 0; k < kMaxCond; ++k) {
            if (k < nc) {
              float fc[8];
              unpack(rec[u][k], fc);
#pragma unroll
              for (int i = 0; i < 8; ++i) fc[i] = convert_param(p, fc[i], fxe[i]);
              combine_packet(q, k, b, pk - b * p.pk_per_sample, g, fc, fu);
            }
          }
          float thr8[8];
          if (clamp) {
            if (p.pk_per_sample != 0) {
              const float tpk = __ldg(p.thr + b);
#pragma unroll
              for (int i = 0; i < 8; ++i) thr8[i] = tpk;
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i) thr8[i] = __ldg(p.thr + (e + i) / p.per_sample);
            }
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) fT[i] = finish_x0(p, g[i], fxe[i], clamp ? thr8[i] : 1.f, clamp);
        }
        Raw<TS> rmo;
        round_pack(rmo, fT);
        if (gmo != nullptr) stg_pk(gmo + e, rmo);
        if (FORM != DPM_FORM_NONE) {
          if (FAST) {
            fast_update8<FORM>(p, fx, fT, fm1, fm2, fo);
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) fo[i] = update_value<FORM>(p, fx[i], fT[i], kM1 ? fm1[i] : 0.f, kM2 ? fm2[i] : 0.f);
          }
          Raw<TS> ro;
          pack(ro, fo);
          stg_pk(go + e, ro);
#pragma unroll
          for (int k = 0; k < kMaxCond; ++k)
            if (k < nc && mp.rep[k] != nullptr) stg_pk(static_cast<TS*>(mp.rep[k]) + e, ro);
        }
      }
    }
  }
}

// generic element-wise variant of k_step_multi_masked (k_step_multi_scalar with the weights)
__global__ void __launch_bounds__(256) k_step_multi_masked_scalar(const __grid_constant__ MaskedParams q) {
  const MultiParams& mpc = q.m;
  KParams p = mpc.k;
  if (p.dev_coef != nullptr) {
    const float* c = p.dev_coef;
    p.a = c[0]; p.c0 = c[1]; p.c1 = c[2]; p.c2 = c[3];
    p.w0 = c[4]; p.w1 = c[5]; p.w2 = c[6]; p.w3 = c[7]; p.w4 = c[8];
    p.alpha_e = c[9]; p.sigma_e = c[10];
    p.fast_div = 0;
  }
  const int sd = p.state_dtype, md = p.model_dtype, nc = mpc.n_cond;
  const FormReads reads = form_reads(p.form);
  const bool clamp = p.thr != nullptr;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (size_t)gridDim.x * blockDim.x) {
    const uint64_t gi = i + p.elem_offset;
    const float x = reads.x ? load_any(p.x, sd, i) : 0.f;
    const float m1 = reads.m1 ? load_any(p.m1, sd, i) : 0.f;
    const float m2 = reads.m2 ? load_any(p.m2, sd, i) : 0.f;
    const float xe = p.use_xe ? ((reads.x && p.xe_is_x) ? x : load_any(p.xe, sd, i)) : 0.f;
    const float eu = convert_param(p, load_any(p.eu, md, i), xe);
    float eps = eu;
    for (int k = 0; k < nc; ++k)
      eps = eps + elem_weight(q, k, gi) * (convert_param(p, load_any(mpc.ec[k], md, i), xe) - eu);
    const float mv = finish_x0(p, eps, xe, clamp ? p.thr[gi / p.per_sample] : 1.f, clamp);
    if (p.m_out) store_any(p.m_out, sd, i, mv);
    const float T0 = round_any(sd, mv);
    float o;
    switch (p.form) {
      case DPM_FORM_LIN1: o = update_value<DPM_FORM_LIN1>(p, x, T0, m1, m2); break;
      case DPM_FORM_LIN2: o = update_value<DPM_FORM_LIN2>(p, x, T0, m1, m2); break;
      case DPM_FORM_LIN3: o = update_value<DPM_FORM_LIN3>(p, x, T0, m1, m2); break;
      case DPM_FORM_DIFF2: o = update_value<DPM_FORM_DIFF2>(p, x, T0, m1, m2); break;
      case DPM_FORM_MS3: o = update_value<DPM_FORM_MS3>(p, x, T0, m1, m2); break;
      case DPM_FORM_SS3T: o = update_value<DPM_FORM_SS3T>(p, x, T0, m1, m2); break;
      default: continue;
    }
    store_any(p.out, sd, i, o);
    for (int k = 0; k < nc; ++k)
      if (mpc.rep[k] != nullptr) store_any(mpc.rep[k], sd, i, o);
  }
}

typedef void (*MaskedKernel)(const MaskedParams);

int launch_step_multi_masked(const MaskedParams& q, const Tuning& t, cudaStream_t stream) {
  const KParams& p = q.m.k;
  for (int k = 0; k < q.m.n_cond; ++k) {   // maps the packets cannot read: the generic kernel
    if (q.w[k] == nullptr) continue;
    const bool vec = q.period[k] % kPacket == 0 && (reinterpret_cast<uintptr_t>(q.w[k]) & 15) == 0;
    if (p.pk_per_sample == 0 || (q.period[k] != 1 && !vec)) return 1;
  }
  const bool fast = fast_path_ok(p);
  MaskedKernel k = with_packet_pair(p.model_dtype, p.state_dtype, [&](auto pair) -> MaskedKernel {
    using TE = typename decltype(pair)::TE;
    using TS = typename decltype(pair)::TS;
    return with_form(p.form, [&](auto form) -> MaskedKernel {
      constexpr int FORM = decltype(form)::value;
      return fast ? k_step_multi_masked<TE, TS, FORM, true> : k_step_multi_masked<TE, TS, FORM, false>;
    });
  });
  if (k == nullptr) return 1;  // other dtype pairs: the generic kernel
  const int threads = t.threads > 0 && t.threads <= kMultiThreads ? t.threads : kMultiThreads;
  const uint64_t tile_pk = (uint64_t)threads * kMultiUnroll;
  const uint64_t tiles = ((uint64_t)p.npk + tile_pk - 1) / tile_pk;
  const uint64_t cap = t.ctas_per_sm > 0 ? (uint64_t)sm_count() * t.ctas_per_sm : tiles;
  const uint32_t grid = (uint32_t)(tiles < cap ? tiles : cap);
  if (grid == 0) return 0;
  cudaError_t le = launch_pdl(k, grid, (unsigned)threads, 0, stream, q);
  if (le != cudaSuccess) return launch_error("masked multi-condition step launch failed", le);
  count_launch();
  return 0;
}

int launch_step_multi_masked_scalar(const MaskedParams& q, cudaStream_t stream) {
  if (q.m.k.n == 0) return 0;
  const int threads = 256;
  const uint64_t blocks = (q.m.k.n + threads - 1) / threads;
  const uint64_t cap = (uint64_t)sm_count() * 8;
  const uint32_t grid = (uint32_t)(blocks < cap ? blocks : cap);
  k_step_multi_masked_scalar<<<grid, threads, 0, stream>>>(q);
  count_launch();
  return 0;
}

// ---- dpm_replicate: x read once, written to `copies` consecutive blocks --------------------------------------------
__global__ void __launch_bounds__(256) k_replicate(const uint4* __restrict__ src, char* __restrict__ dst, uint64_t words,
                                                   uint64_t bytes, int copies) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (uint64_t)gridDim.x * blockDim.x) {
    uint4 v;
    asm volatile("ld.global.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i));
    for (int c = 0; c < copies; ++c) {
      uint4* d = reinterpret_cast<uint4*>(dst + (uint64_t)c * bytes) + i;
      asm volatile("st.global.L1::no_allocate.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(d), "r"(v.x), "r"(v.y), "r"(v.z),
                   "r"(v.w) : "memory");
    }
  }
}

int launch_replicate(void* dst, const void* src, uint64_t bytes, int copies, cudaStream_t stream) {
  if (bytes == 0) return 0;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(dst) || !al16(src) || (bytes & 15) != 0) return 1;
  const uint64_t words = bytes / 16;
  const uint64_t blocks = (words + 255) / 256;
  const uint64_t cap = (uint64_t)sm_count() * 16;
  const uint32_t grid = (uint32_t)(blocks < cap ? blocks : cap);
  k_replicate<<<grid, 256, 0, stream>>>(static_cast<const uint4*>(src), static_cast<char*>(dst), words, bytes, copies);
  count_launch();
  return 0;
}

}  // namespace dpm
