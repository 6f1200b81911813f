// step_direct.cu -- variant 0: one tile per CTA (a persistent grid when ctas_per_sm is set), 128/256-bit global
// loads straight to registers.
//
// One thread owns kUnroll packets of 8 consecutive elements per tile; all loads of a tile are
// issued before the first use so that (streams x kUnroll) 16/32-byte requests are in flight per
// thread. HBM-bound: (k+2)*s algorithmic bytes per element for a pure order-k update.
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kUnroll = 2;
constexpr int kMaxThreads = 512;

// FAST: the straight-line packet code of common.cuh (fast_model8 / fast_update8; launch-time test
// fast_path_ok). FAST = false keeps every parameterisation, per-element thresholds and IEEE divisions.
// RND (only with FAST = false): reference-rounding mode (dpm_step_desc.raw_round) on the vector path -- the 16-bit
// CFG combine (three rounded ops) and the rounded differences of raw 16-bit buffers, per element, between 128/256-bit
// loads and stores.
// RS (only with NE == 2 and RND = false): guidance rescale (dpm_step_rescaled) with the per-sample ratio p.ratio, read
// like the per-sample thresholds.
// PG (only with NE == 2, RND = false and RS = false): per-sample guidance (dpm_step_guided) with the scale p.gscale
// and, when p.ratio is set, the rescale -- one kernel family for rescale on and off. With FAST = false it also serves
// CFG-Zero* (dpm_step_cfgzero: p.zs set, p.gscale NULL for one scale p.guidance) and TCFG (dpm_step_tcfg: p.td set,
// likewise).
// APG (only with NE == 2, FAST = false and no other option; the kernel k_step_direct_apg): adaptive projected guidance
// (dpm_step_apg) with the per-sample words p.apg_a / p.apg_b; reads the fp32 direction p.apg_r in place of e_uncond
// when it is set.
template <typename TE, typename TS, int NE, int FORM, bool FAST, bool RND, bool RS, bool PG, bool APG>
__device__ __forceinline__ void step_direct_body(const KParams& p) {
  constexpr bool kX = form_reads(FORM).x, kM1 = form_reads(FORM).m1, kM2 = form_reads(FORM).m2;
  const TS* __restrict__ gx = static_cast<const TS*>(p.x);
  const TS* __restrict__ gxe = static_cast<const TS*>(p.xe);
  const TS* __restrict__ gm0 = static_cast<const TS*>(p.m0);
  const TS* __restrict__ gm1 = static_cast<const TS*>(p.m1);
  const TS* __restrict__ gm2 = static_cast<const TS*>(p.m2);
  const TE* __restrict__ gec = static_cast<const TE*>(p.ec);
  const TE* __restrict__ geu = static_cast<const TE*>(p.eu);
  TS* __restrict__ gmo = static_cast<TS*>(p.m_out);
  TS* __restrict__ go = static_cast<TS*>(p.out);
  TS* __restrict__ go2 = static_cast<TS*>(p.out2);

  const uint32_t npk = p.npk;
  const uint32_t tile_pk = blockDim.x * kUnroll;
  const bool sep_xe = (NE > 0) && p.use_xe && !(kX && p.xe_is_x);
  const bool clamp = (NE > 0) && (p.thr != nullptr);
  const bool apg_r = APG && p.apg_r != nullptr;
  pdl_trigger();
  pdl_wait();

  for (uint64_t tile0 = (uint64_t)blockIdx.x * tile_pk; tile0 < npk;
       tile0 += (uint64_t)gridDim.x * tile_pk) {
    Raw<TS> rx[kUnroll], rxe[kUnroll], rm0[kUnroll], rm1[kUnroll], rm2[kUnroll];
    Raw<TE> rec[kUnroll], reu[kUnroll];
    Raw<float> rr[APG ? kUnroll : 1];
    // ---- issue every load of the tile ----
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        if (kX) ldg_pk(rx[u], gx + e);
        if (NE > 0) {
          ldg_pk(rec[u], gec + e);
          if constexpr (APG) {
            if (apg_r) ldg_pk(rr[u], p.apg_r + e);
            else ldg_pk(reu[u], geu + e);
          } else if (NE == 2) {
            ldg_pk(reu[u], geu + e);
          }
          if (sep_xe) ldg_pk(rxe[u], gxe + e);
        } else {
          ldg_pk(rm0[u], gm0 + e);
        }
        if (kM1) ldg_pk(rm1[u], gm1 + e);
        if (kM2) ldg_pk(rm2[u], gm2 + e);
      }
    }
    // ---- compute + store ----
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        float fx[8], fxe[8], fT[8], fm1[8], fm2[8], fo[8];
        if (kX) unpack(rx[u], fx);
        if (kM1) unpack(rm1[u], fm1);
        if (kM2) unpack(rm2[u], fm2);
        if (NE > 0 && FAST) {
          float fec[8], feu[8];
          unpack(rec[u], fec);
          if (NE == 2) unpack(reu[u], feu);
          const float s_thr = clamp ? __ldg(p.thr + (uint32_t)pk / p.pk_per_sample) : 1.f;   // packet index < 2^32 (npk)
          if constexpr (PG) {
            const float r = p.ratio != nullptr ? __ldg(p.ratio + (uint32_t)pk / p.pk_per_sample) : 1.f;
            const float gs = __ldg(p.gscale + (uint32_t)pk / p.pk_per_sample);
            if (sep_xe) {
              unpack(rxe[u], fxe);
              fast_model8<NE, false, true>(p, fxe, fec, feu, clamp, s_thr, fT, r, gs);
            } else {
              fast_model8<NE, false, true>(p, fx, fec, feu, clamp, s_thr, fT, r, gs);   // fx: as below
            }
          } else {
            const float r = RS ? __ldg(p.ratio + (uint32_t)pk / p.pk_per_sample) : 1.f;
            if (sep_xe) {
              unpack(rxe[u], fxe);
              fast_model8<NE, RS>(p, fxe, fec, feu, clamp, s_thr, fT, r);
            } else {
              fast_model8<NE, RS>(p, fx, fec, feu, clamp, s_thr, fT, r);   // fx is only read when the conversion needs it (then it is loaded)
            }
          }
          Raw<TS> rmo;
          round_pack(rmo, fT);
          if (gmo != nullptr) stg_pk(gmo + e, rmo);
        } else if (NE > 0) {
          float fec[8], feu[8];
          unpack(rec[u], fec);
          if constexpr (APG) {
            if (apg_r) unpack(rr[u], feu);
            else unpack(reu[u], feu);
          } else if (NE == 2) {
            unpack(reu[u], feu);
          }
          if (sep_xe) {
            unpack(rxe[u], fxe);
          } else if (kX) {
#pragma unroll
            for (int i = 0; i < 8; ++i) fxe[i] = fx[i];
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) fxe[i] = 0.f;
          }
          if constexpr (APG) {
            // samples hold whole packets here (pick_direct): the sample's words, bypass and threshold are one scalar each
            const uint32_t b = (uint32_t)(pk / p.pk_per_sample);
            const float A = __ldg(p.apg_a + b), B = __ldg(p.apg_b + b);
            const bool bypass = p.gscale != nullptr && __ldg(p.gscale + b) == 1.f;
            const float tpk = clamp ? __ldg(p.thr + b) : 1.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) fT[i] = apg_value(p, fxe[i], fec[i], feu[i], apg_r, A, B, bypass, tpk, clamp);
          } else if constexpr (PG) {
            // samples hold whole packets here (pick_direct): the sample's scale, ratio (when the launch is rescaled) and
            // threshold are one scalar each per packet
            const uint32_t b = (uint32_t)(pk / p.pk_per_sample);
            const float gpk = p.gscale != nullptr ? __ldg(p.gscale + b) : p.guidance;
            const float rpk = p.zs != nullptr ? __ldg(p.zs + b) : (p.ratio != nullptr ? __ldg(p.ratio + b) : 1.f);
            const float tpk = clamp ? __ldg(p.thr + b) : 1.f;
            // the kind of the combine is uniform per packet: one branch per packet, straight-line code per element
            auto guided8 = [&](auto kind, float r, float r2) {
#pragma unroll
              for (int i = 0; i < 8; ++i)
                fT[i] = model_value<NE, false, false, decltype(kind)::value>(p, fxe[i], fec[i], feu[i], tpk, clamp,
                                                                             r, gpk, r2);
            };
            const int kind = pg_kind(p, gpk);
            if (kind == kPgBypass) guided8(std::integral_constant<int, kPgBypass>{}, rpk, 0.f);
            else if (kind == kPgRescale) guided8(std::integral_constant<int, kPgRescale>{}, rpk, 0.f);
            else if (kind == kPgZeroStar) guided8(std::integral_constant<int, kPgZeroStar>{}, rpk, 0.f);
            else if (kind == kPgTangential)   // TCFG's two words, loaded where they are used
              guided8(std::integral_constant<int, kPgTangential>{}, __ldg(p.td + 2 * b), __ldg(p.td + 2 * b + 1));
            else guided8(std::integral_constant<int, kPgCombine>{}, rpk, 0.f);
          } else {
            float thr8[8];
            const bool thr_uniform = p.pk_per_sample != 0;
            if (clamp) {
              if (thr_uniform) {
                const float tpk = __ldg(p.thr + (uint32_t)(pk / p.pk_per_sample));
#pragma unroll
                for (int i = 0; i < 8; ++i) thr8[i] = tpk;
              } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) thr8[i] = __ldg(p.thr + (e + i) / p.per_sample);
              }
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i) thr8[i] = 1.f;
            }
            float r8[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) r8[i] = 1.f;
            if (RS) {
              if (thr_uniform) {
                const float rpk = __ldg(p.ratio + (uint32_t)(pk / p.pk_per_sample));
#pragma unroll
                for (int i = 0; i < 8; ++i) r8[i] = rpk;
              } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) r8[i] = __ldg(p.ratio + (e + i) / p.per_sample);
              }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
              fT[i] = model_value<NE, RND, RS>(p, fxe[i], fec[i], NE == 2 ? feu[i] : 0.f, thr8[i], clamp, r8[i]);
          }
          Raw<TS> rmo;
          round_pack(rmo, fT);
          if (gmo != nullptr) stg_pk(gmo + e, rmo);
        } else {
          unpack(rm0[u], fT);
        }
        if (FORM != DPM_FORM_NONE) {
          if (FAST) {
            fast_update8<FORM>(p, fx, fT, fm1, fm2, fo);
          } else {
#pragma unroll
            for (int i = 0; i < 8; ++i)
              fo[i] = update_value<FORM, RND>(p, fx[i], fT[i], kM1 ? fm1[i] : 0.f,
                                              kM2 ? fm2[i] : 0.f);
          }
          Raw<TS> ro;
          pack(ro, fo);
          stg_pk(go + e, ro);
          if (go2 != nullptr) stg_pk(go2 + e, ro);
        }
      }
    }
  }
}

template <typename TE, typename TS, int NE, int FORM, bool FAST, bool RND = false, bool RS = false, bool PG = false>
__global__ void __launch_bounds__(kMaxThreads) k_step_direct(const __grid_constant__ KParams p) {
  step_direct_body<TE, TS, NE, FORM, FAST, RND, RS, PG, false>(p);
}
template <typename TE, typename TS, int FORM>
__global__ void __launch_bounds__(kMaxThreads) k_step_direct_apg(const __grid_constant__ KParams p) {
  step_direct_body<TE, TS, 2, FORM, false, false, false, false, true>(p);
}

// ---- fully generic element-wise kernel: any dtype mix, any alignment, tails ------------------
// RND = true: reference-rounding mode (common.cuh) for the launches the <RND> vector kernels do not serve:
// unaligned views, tails and fp32 network outputs.
// RS = true: guidance rescale (n_model == 2) for unaligned views, tails and dev_coef launches.
// PG = true: per-sample guidance (n_model == 2; rescale iff p.ratio is set), CFG-Zero* (p.zs set) and TCFG (p.td set),
// likewise.
// APG = true (the kernel k_step_scalar_apg): adaptive projected guidance (n_model == 2), likewise.
template <bool RND, bool RS, bool PG, bool APG>
__device__ __forceinline__ void step_scalar_body(const KParams& pc) {
  KParams p = pc;
  if (pc.dev_coef != nullptr) {
    // scalars produced on the device by the adaptive controller (adaptive_ctl.cu: CO_* layout)
    const float* c = pc.dev_coef;
    p.a = c[0]; p.c0 = c[1]; p.c1 = c[2]; p.c2 = c[3];
    p.w0 = c[4]; p.w1 = c[5]; p.w2 = c[6]; p.w3 = c[7]; p.w4 = c[8];
    p.alpha_e = c[9]; p.sigma_e = c[10];
    p.fast_div = 0;
    if (APG) { p.apg_alpha = c[9]; p.apg_sigma = c[10]; }   // (no EDM launch takes dev_coef: the marginals)
  }
  const int sd = p.state_dtype, md = p.model_dtype;
  const FormReads reads = form_reads(p.form);
  const bool need_x = reads.x, need_m1 = reads.m1, need_m2 = reads.m2;
  const bool clamp = p.n_model > 0 && p.thr != nullptr;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n;
       i += (size_t)gridDim.x * blockDim.x) {
    float x = need_x ? load_any(p.x, sd, i) : 0.f;
    float m1 = need_m1 ? load_any(p.m1, sd, i) : 0.f;
    float m2 = need_m2 ? load_any(p.m2, sd, i) : 0.f;
    float T0;
    if (p.n_model > 0) {
      float xe = p.use_xe ? ((need_x && p.xe_is_x) ? x : load_any(p.xe, sd, i)) : 0.f;
      float ec = load_any(p.ec, md, i);
      const bool apg_r = APG && p.apg_r != nullptr;
      float eu = p.n_model == 2 && !apg_r ? load_any(p.eu, md, i) : 0.f;
      float thr = clamp ? p.thr[(i + p.elem_offset) / p.per_sample] : 1.f;
      float mv;
      if constexpr (APG) {
        const uint64_t b = (i + p.elem_offset) / p.per_sample;
        const bool bypass = p.gscale != nullptr && p.gscale[b] == 1.f;
        mv = apg_value(p, xe, ec, apg_r ? p.apg_r[i + p.elem_offset] : eu, apg_r, p.apg_a[b], p.apg_b[b], bypass, thr,
                       clamp);
      } else if constexpr (PG) {
        const uint64_t b = (i + p.elem_offset) / p.per_sample;
        const float r = p.zs != nullptr ? p.zs[b]
                        : (p.td != nullptr ? p.td[2 * b] : (p.ratio != nullptr ? p.ratio[b] : 1.f));
        mv = model_value<2, false, false, kPgAny>(p, xe, ec, eu, thr, clamp, r,
                                                  p.gscale != nullptr ? p.gscale[b] : p.guidance,
                                                  p.td != nullptr ? p.td[2 * b + 1] : 0.f);
      } else if (RS) {
        mv = model_value<2, false, true>(p, xe, ec, eu, thr, clamp, p.ratio[(i + p.elem_offset) / p.per_sample]);
      } else {
        mv = p.n_model == 2 ? model_value<2, RND>(p, xe, ec, eu, thr, clamp)
                            : model_value<1, RND>(p, xe, ec, eu, thr, clamp);
      }
      T0 = round_any(sd, mv);
      if (p.m_out) store_any(p.m_out, sd, i, mv);
    } else {
      T0 = load_any(p.m0, sd, i);
    }
    float o;
    switch (p.form) {
      case DPM_FORM_LIN1: o = update_value<DPM_FORM_LIN1, RND>(p, x, T0, m1, m2); break;
      case DPM_FORM_LIN2: o = update_value<DPM_FORM_LIN2, RND>(p, x, T0, m1, m2); break;
      case DPM_FORM_LIN3: o = update_value<DPM_FORM_LIN3, RND>(p, x, T0, m1, m2); break;
      case DPM_FORM_DIFF2: o = update_value<DPM_FORM_DIFF2, RND>(p, x, T0, m1, m2); break;
      case DPM_FORM_MS3: o = update_value<DPM_FORM_MS3, RND>(p, x, T0, m1, m2); break;
      case DPM_FORM_SS3T: o = update_value<DPM_FORM_SS3T, RND>(p, x, T0, m1, m2); break;
      default: continue;
    }
    store_any(p.out, sd, i, o);
    if (p.out2) store_any(p.out2, sd, i, o);
  }
}

template <bool RND, bool RS = false, bool PG = false>
__global__ void __launch_bounds__(256) k_step_scalar(const __grid_constant__ KParams pc) {
  step_scalar_body<RND, RS, PG, false>(pc);
}
__global__ void __launch_bounds__(256) k_step_scalar_apg(const __grid_constant__ KParams pc) {
  step_scalar_body<false, false, false, true>(pc);
}

// ---- dispatch ---------------------------------------------------------------------------------
typedef void (*StepKernel)(const KParams);

// FAST: NE == 0 has no model conversion, so there only SS3T (division by w4) has a <FAST = false> twin.
// RND: an fp32 state with raw network outputs in bf16 / f16 (NE >= 1), or fp32 buffers holding such raw outputs
// (NE == 0, differences rounded).
// RS: guidance rescale, NE == 2 only (the C-ABI rejects it together with raw_round).
// PG: per-sample guidance, NE == 2 only; serves rescaled and plain launches alike (so it is tested before RS).
// APG: adaptive projected guidance, NE == 2 only, on the IEEE-division instantiations (tested first: it carries gscale
// for its bypass).
// CFG-Zero* (p.zs) and TCFG (p.td): the <PG> instantiations with FAST = false, with or without per-sample scales.
static StepKernel pick_direct(const KParams& p) {
  const bool zs = p.zs != nullptr || p.td != nullptr;
  const bool fast = fast_path_ok(p) && !zs, rnd = p.raw_round != 0, rs = p.ratio != nullptr;
  const bool pg = p.gscale != nullptr || zs;
  const bool apg = p.apg_a != nullptr;
  if ((pg || apg) && p.pk_per_sample == 0) return nullptr;
  return pick_step<StepKernel>(p, [&](auto pair, auto ne, auto form) -> StepKernel {
    using TE = typename decltype(pair)::TE;
    using TS = typename decltype(pair)::TS;
    constexpr int NE = decltype(ne)::value, FORM = decltype(form)::value;
    if (apg) {   // samples that do not hold whole packets: the generic kernel (k_step_scalar_apg)
      if constexpr (NE == 2)
        return k_step_direct_apg<TE, TS, FORM>;
      else
        return nullptr;
    }
    if (pg) {   // samples that do not hold whole packets: the generic kernel (k_step_scalar<PG>)
      if constexpr (NE == 2)
        return fast ? k_step_direct<TE, TS, 2, FORM, true, false, false, true>
                    : k_step_direct<TE, TS, 2, FORM, false, false, false, true>;
      else
        return nullptr;
    }
    if (rs) {
      if constexpr (NE == 2)
        return fast ? k_step_direct<TE, TS, 2, FORM, true, false, true> : k_step_direct<TE, TS, 2, FORM, false, false, true>;
      else
        return nullptr;
    }
    if (rnd) {
      if constexpr (std::is_same_v<TS, float> && (NE == 0) == std::is_same_v<TE, float>)
        return k_step_direct<TE, TS, NE, FORM, false, true>;
      else
        return nullptr;
    }
    if constexpr (NE == 0 && FORM != DPM_FORM_SS3T)
      return k_step_direct<TE, TS, NE, FORM, true>;
    else
      return fast ? k_step_direct<TE, TS, NE, FORM, true> : k_step_direct<TE, TS, NE, FORM, false>;
  });
}

int launch_step_direct(const KParams& p, const Tuning& t, cudaStream_t stream) {
  StepKernel k = pick_direct(p);
  if (k == nullptr) return 1;  // not served here
  const int threads = t.threads > 0 ? t.threads : 256;
  const uint32_t tile_pk = (uint32_t)threads * kUnroll;
  uint64_t tiles = ((uint64_t)p.npk + tile_pk - 1) / tile_pk;
  // Default: one tile per CTA, as many waves as it takes. The block scheduler hands a freed slot the next tile, so
  // the HBM queues stay full to the end of the launch; on H100 this streams c2's steps 6 % faster than any
  // persistent grid (SMs x 4..32 CTAs, DESIGN.md §4). ctas_per_sm > 0 caps the grid at SMs x ctas_per_sm instead
  // (the kernel's tile loop then strides over the grid).
  uint64_t cap = t.ctas_per_sm > 0 ? (uint64_t)sm_count() * t.ctas_per_sm : tiles;
  uint32_t grid = (uint32_t)(tiles < cap ? tiles : cap);
  if (grid == 0) return 0;
  cudaError_t le = launch_pdl(k, grid, (unsigned)threads, 0, stream, p);
  if (le != cudaSuccess) return launch_error("step launch failed", le);
  count_launch();
  return 0;
}

int launch_step_scalar(const KParams& p, cudaStream_t stream) {
  if (p.n == 0) return 0;
  const int threads = 256;
  uint64_t blocks = (p.n + threads - 1) / threads;
  uint64_t cap = (uint64_t)sm_count() * 8;
  uint32_t grid = (uint32_t)(blocks < cap ? blocks : cap);
  if (p.raw_round) k_step_scalar<true><<<grid, threads, 0, stream>>>(p);
  else if (p.apg_a) k_step_scalar_apg<<<grid, threads, 0, stream>>>(p);
  else if (p.gscale || p.zs || p.td) k_step_scalar<false, false, true><<<grid, threads, 0, stream>>>(p);
  else if (p.ratio) k_step_scalar<false, true><<<grid, threads, 0, stream>>>(p);
  else k_step_scalar<false><<<grid, threads, 0, stream>>>(p);
  count_launch();
  return 0;
}

}  // namespace dpm
