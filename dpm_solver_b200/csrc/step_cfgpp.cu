// step_cfgpp.cu -- CFG++ (Chung, Kim, Park, Nam and Ye, ICLR 2025, arXiv:2406.08070) fused into the DPM-Solver++ order-1
// and multistep order-2 updates (dpm_step_cfgpp).
//
// CFG++ denoises with the guided data prediction and re-noises with the UNCONDITIONAL noise. Per element, in fp32 with
// every op rounded:
//   U = round_S(T_u)   T_u: the x0 the unguided step buffers for e_u alone (model_value<1> / fast_model8<1>)
//   G = round_S(T_g)   T_g: the x0 the CFG step buffers for (e_c, e_u) with the sample's scale (a per-sample scale of 1
//                           takes e_c, a scalar scale is always combined)
//   d = G - U
//   LIN1:  out = (a*x + c0*U) + g*d
//   DIFF2: out = ((a*x + c0*U) + g*d) + c1*(w0*(G - m1))        (m1: the previous step's U)
// with g = alpha_t. m_out receives U (what the multistep solver buffers), out2 a second copy of out (the doubled network
// input). Algorithmic traffic: x, e_c, e_u [, m1] read, out, out2, m_out written -- 6s (LIN1) / 7s (DIFF2) bytes per
// element, those of the plain CFG step.
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kCfgppUnroll = 2;
constexpr int kCfgppThreads = 512;

// the update of the contract above, one element (U and G as they read back from the state type)
template <int FORM>
__device__ __forceinline__ float cfgpp_update(const CfgppParams& q, float x, float U, float G, float m1) {
  const KParams& p = q.k;
  const float o = (p.a * x + p.c0 * U) + q.g * (G - U);
  if (FORM == DPM_FORM_DIFF2) return o + p.c1 * (p.w0 * (G - m1));
  return o;
}

// FAST: NOISE (exact constant division), FLOW or EDM networks (fast_path_ok); the two values by the packet code of
// common.cuh. FAST = false: every parameterisation and IEEE division, per element by model_value.
// Per-sample scales need samples that hold whole packets (pk_per_sample != 0); the host routes other launches to
// k_step_cfgpp_scalar.
template <typename TE, typename TS, int FORM, bool FAST>
__global__ void __launch_bounds__(kCfgppThreads) k_step_cfgpp(const __grid_constant__ CfgppParams q) {
  const KParams& p = q.k;
  constexpr bool kM1 = FORM == DPM_FORM_DIFF2;
  const TS* __restrict__ gx = static_cast<const TS*>(p.x);
  const TS* __restrict__ gxe = static_cast<const TS*>(p.xe);
  const TS* __restrict__ gm1 = static_cast<const TS*>(p.m1);
  const TE* __restrict__ gec = static_cast<const TE*>(p.ec);
  const TE* __restrict__ geu = static_cast<const TE*>(p.eu);
  TS* __restrict__ gmo = static_cast<TS*>(p.m_out);
  TS* __restrict__ go = static_cast<TS*>(p.out);
  TS* __restrict__ go2 = static_cast<TS*>(p.out2);

  const uint32_t npk = p.npk;
  const uint32_t tile_pk = blockDim.x * kCfgppUnroll;
  const bool sep_xe = !p.xe_is_x;
  const bool per_sample = p.gscale != nullptr;
  pdl_trigger();
  pdl_wait();

  for (uint64_t tile0 = (uint64_t)blockIdx.x * tile_pk; tile0 < npk; tile0 += (uint64_t)gridDim.x * tile_pk) {
    Raw<TS> rx[kCfgppUnroll], rxe[kCfgppUnroll], rm1[kCfgppUnroll];
    Raw<TE> rec[kCfgppUnroll], reu[kCfgppUnroll];
    // ---- issue every load of the tile ----
#pragma unroll
    for (int u = 0; u < kCfgppUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        ldg_pk(rx[u], gx + e);
        ldg_pk(rec[u], gec + e);
        ldg_pk(reu[u], geu + e);
        if (sep_xe) ldg_pk(rxe[u], gxe + e);
        if (kM1) ldg_pk(rm1[u], gm1 + e);
      }
    }
    // ---- compute + store ----
#pragma unroll
    for (int u = 0; u < kCfgppUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        float fx[8], fxe[8], fm1[8], fec[8], feu[8], fG[8], fo[8];
        unpack(rx[u], fx);
        if (kM1) unpack(rm1[u], fm1);
        unpack(rec[u], fec);
        unpack(reu[u], feu);
        if (sep_xe) {
          unpack(rxe[u], fxe);
        } else {
#pragma unroll
          for (int i = 0; i < 8; ++i) fxe[i] = fx[i];
        }
        // the sample's scale: one scalar per packet (samples hold whole packets here)
        const float gs = per_sample ? __ldg(p.gscale + (uint32_t)pk / p.pk_per_sample) : p.guidance;
        if (FAST) {
          // G first: fast_model8 converts a FLOW / EDM pair in place, so feu then holds the converted e_u, and
          // fast_finish8 completes U exactly as fast_model8<1> would for e_u alone (eps -> x0 of a NOISE output)
          if (per_sample) fast_model8<2, false, true>(p, fxe, fec, feu, false, 1.f, fG, 1.f, gs);
          else fast_model8<2>(p, fxe, fec, feu, false, 1.f, fG);
          fast_finish8(p, fxe, false, 1.f, feu);
        } else {
          const bool bypass = per_sample && gs == 1.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            fG[i] = bypass ? model_value<2, false, false, kPgBypass>(p, fxe[i], fec[i], feu[i], 1.f, false, 1.f, gs)
                           : model_value<2, false, false, kPgCombine>(p, fxe[i], fec[i], feu[i], 1.f, false, 1.f, gs);
            feu[i] = model_value<1>(p, fxe[i], feu[i], 0.f, 1.f, false);
          }
        }
        Raw<TS> rmo, rg;
        round_pack(rmo, feu);   // U, as the buffer reads it back
        round_pack(rg, fG);     // G likewise
        if (gmo != nullptr) stg_pk(gmo + e, rmo);
#pragma unroll
        for (int i = 0; i < 8; ++i) fo[i] = cfgpp_update<FORM>(q, fx[i], feu[i], fG[i], kM1 ? fm1[i] : 0.f);
        Raw<TS> ro;
        pack(ro, fo);
        stg_pk(go + e, ro);
        if (go2 != nullptr) stg_pk(go2 + e, ro);
      }
    }
  }
}

// generic element-wise variant: any dtype pair, any alignment, tails, samples that do not hold whole packets
__global__ void __launch_bounds__(256) k_step_cfgpp_scalar(const __grid_constant__ CfgppParams q) {
  const KParams& p = q.k;
  const int sd = p.state_dtype, md = p.model_dtype;
  const bool diff2 = p.form == DPM_FORM_DIFF2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (size_t)gridDim.x * blockDim.x) {
    const float x = load_any(p.x, sd, i);
    const float m1 = diff2 ? load_any(p.m1, sd, i) : 0.f;
    const float xe = p.xe_is_x ? x : load_any(p.xe, sd, i);
    const float ec = load_any(p.ec, md, i), eu = load_any(p.eu, md, i);
    const float gs = p.gscale != nullptr ? p.gscale[(i + p.elem_offset) / p.per_sample] : p.guidance;
    const float G = round_any(sd, p.gscale != nullptr && gs == 1.f
                                      ? model_value<2, false, false, kPgBypass>(p, xe, ec, eu, 1.f, false, 1.f, gs)
                                      : model_value<2, false, false, kPgCombine>(p, xe, ec, eu, 1.f, false, 1.f, gs));
    const float U = model_value<1>(p, xe, eu, 0.f, 1.f, false);
    const float Ur = p.m_out ? store_any(p.m_out, sd, i, U) : round_any(sd, U);
    const float o = diff2 ? cfgpp_update<DPM_FORM_DIFF2>(q, x, Ur, G, m1) : cfgpp_update<DPM_FORM_LIN1>(q, x, Ur, G, m1);
    store_any(p.out, sd, i, o);
    if (p.out2) store_any(p.out2, sd, i, o);
  }
}

typedef void (*CfgppKernel)(const CfgppParams);

int launch_step_cfgpp(const CfgppParams& q, const Tuning& t, cudaStream_t stream) {
  const KParams& p = q.k;
  if (p.gscale != nullptr && p.pk_per_sample == 0) return 1;   // per-sample scales by element: the generic kernel
  const bool fast = fast_path_ok(p);
  CfgppKernel k = with_packet_pair(p.model_dtype, p.state_dtype, [&](auto pair) -> CfgppKernel {
    using TE = typename decltype(pair)::TE;
    using TS = typename decltype(pair)::TS;
    if (p.form == DPM_FORM_LIN1)
      return fast ? k_step_cfgpp<TE, TS, DPM_FORM_LIN1, true> : k_step_cfgpp<TE, TS, DPM_FORM_LIN1, false>;
    return fast ? k_step_cfgpp<TE, TS, DPM_FORM_DIFF2, true> : k_step_cfgpp<TE, TS, DPM_FORM_DIFF2, false>;
  });
  if (k == nullptr) return 1;  // other dtype pairs: the generic kernel
  const int threads = t.threads > 0 ? t.threads : 256;
  const uint64_t tile_pk = (uint64_t)threads * kCfgppUnroll;
  const uint64_t tiles = ((uint64_t)p.npk + tile_pk - 1) / tile_pk;
  const uint64_t cap = t.ctas_per_sm > 0 ? (uint64_t)sm_count() * t.ctas_per_sm : tiles;
  const uint32_t grid = (uint32_t)(tiles < cap ? tiles : cap);
  if (grid == 0) return 0;
  cudaError_t le = launch_pdl(k, grid, (unsigned)threads, 0, stream, q);
  if (le != cudaSuccess) return launch_error("cfg++ step launch failed", le);
  count_launch();
  return 0;
}

int launch_step_cfgpp_scalar(const CfgppParams& q, cudaStream_t stream) {
  if (q.k.n == 0) return 0;
  const int threads = 256;
  const uint64_t blocks = (q.k.n + threads - 1) / threads;
  const uint64_t cap = (uint64_t)sm_count() * 8;
  const uint32_t grid = (uint32_t)(blocks < cap ? blocks : cap);
  k_step_cfgpp_scalar<<<grid, threads, 0, stream>>>(q);
  count_launch();
  return 0;
}

}  // namespace dpm
