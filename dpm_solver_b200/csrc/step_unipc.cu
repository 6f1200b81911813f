// step_unipc.cu -- UniPC (Zhao et al. 2023) multistep: the corrector of step i and the predictor of step i+1 in one
// launch per network evaluation (dpm_step_unipc, include/dpm_solver_b200.h).
//
// Per element, with x~ = x~_i (the network input of evaluation i) and m_i its converted model value:
//   x_i      = x~ [+ cd[0]*(m_{i-2} - m_{i-1}) [+ cd[1]*(m_{i-3} - m_{i-1})]] + ct*(m_i - m_{i-1})          (pc > 0)
//   x_i      = x~                                                                                         (pc = 0)
//   x_i rounded to the state dtype in registers
//   x~_{i+1} = a*x_i + c0*m_i [+ cp[0]*(m_{i-1} - m_i) [+ cp[1]*(m_{i-2} - m_i)]]                       (pp > 0)
// differences first, then the sums left to right, each op rounded (-fmad=false). The corrected state never leaves
// registers unless out_c asks for it. Algorithmic traffic of UniPC-2 with a noise network and no CFG: x~, eps, m_{i-1},
// m_{i-2} read, m_i and x~_{i+1} written: 6*s bytes per element.
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kUniUnroll = 2;
constexpr int kUniThreads = 256;

// corrector and predictor of one element (fx: x~_i, T: m_i, m1..m3: m_{i-1..i-3}); returns x~_{i+1}, xc = x_i
template <typename TS>
__device__ __forceinline__ float unipc_value(const UniParams& u, float fx, float T, float m1, float m2, float m3,
                                             float& xc) {
  float c = fx;
  if (u.pc > 0) {
    if (u.pc >= 2) c = c + u.cd[0] * (m2 - m1);
    if (u.pc >= 3) c = c + u.cd[1] * (m3 - m1);
    c = c + u.ct * (T - m1);
    c = round_storage<TS>(c);
  }
  xc = c;
  float o = u.a * c + u.c0 * T;
  if (u.pp >= 2) o = o + u.cp[0] * (m1 - T);
  if (u.pp >= 3) o = o + u.cp[1] * (m2 - T);
  return o;
}

// FAST: param == NOISE, FLOW or EDM, exact constant division, a clamp threshold uniform per packet (fast_path_ok);
// FAST = false: every parameterisation, per-element thresholds, IEEE division. NE == 0 reads m_i from k.m0.
template <typename TE, typename TS, int NE, bool FAST>
__global__ void __launch_bounds__(kUniThreads) k_step_unipc(const __grid_constant__ UniParams up) {
  const KParams& p = up.k;
  const TS* __restrict__ gx = static_cast<const TS*>(p.x);
  const TS* __restrict__ gm0 = static_cast<const TS*>(p.m0);
  const TS* __restrict__ gm1 = static_cast<const TS*>(p.m1);
  const TS* __restrict__ gm2 = static_cast<const TS*>(p.m2);
  const TS* __restrict__ gm3 = static_cast<const TS*>(up.m3);
  const TE* __restrict__ gec = static_cast<const TE*>(p.ec);
  const TE* __restrict__ geu = static_cast<const TE*>(p.eu);
  TS* __restrict__ gmo = static_cast<TS*>(p.m_out);
  TS* __restrict__ go = static_cast<TS*>(p.out);
  TS* __restrict__ go2 = static_cast<TS*>(p.out2);
  TS* __restrict__ goc = static_cast<TS*>(up.out_c);
  const UniReads rd = uni_reads(up.pc, up.pp);
  const bool clamp = (NE > 0) && (p.thr != nullptr);

  const uint32_t npk = p.npk;
  const uint32_t tile_pk = blockDim.x * kUniUnroll;
  pdl_trigger();
  pdl_wait();

  for (uint64_t tile0 = (uint64_t)blockIdx.x * tile_pk; tile0 < npk; tile0 += (uint64_t)gridDim.x * tile_pk) {
    Raw<TS> rx[kUniUnroll], rm0[kUniUnroll], rm1[kUniUnroll], rm2[kUniUnroll], rm3[kUniUnroll];
    Raw<TE> rec[kUniUnroll], reu[kUniUnroll];
#pragma unroll
    for (int u = 0; u < kUniUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        ldg_pk(rx[u], gx + e);
        if (NE > 0) {
          ldg_pk(rec[u], gec + e);
          if (NE == 2) ldg_pk(reu[u], geu + e);
        } else {
          ldg_pk(rm0[u], gm0 + e);
        }
        if (rd.m1) ldg_pk(rm1[u], gm1 + e);
        if (rd.m2) ldg_pk(rm2[u], gm2 + e);
        if (rd.m3) ldg_pk(rm3[u], gm3 + e);
      }
    }
#pragma unroll
    for (int u = 0; u < kUniUnroll; ++u) {
      const uint64_t pk = tile0 + (uint64_t)u * blockDim.x + threadIdx.x;
      if (pk < npk) {
        const size_t e = (size_t)pk * kPacket;
        float fx[8], fT[8], fm1[8], fm2[8], fm3[8], fo[8], fc[8];
        unpack(rx[u], fx);
#pragma unroll
        for (int i = 0; i < 8; ++i) fm1[i] = fm2[i] = fm3[i] = 0.f;
        if (rd.m1) unpack(rm1[u], fm1);
        if (rd.m2) unpack(rm2[u], fm2);
        if (rd.m3) unpack(rm3[u], fm3);
        if (NE > 0) {
          float fec[8], feu[8];
          unpack(rec[u], fec);
          if (NE == 2) unpack(reu[u], feu);
          if (FAST) {
            const float s_thr = clamp ? __ldg(p.thr + (uint32_t)pk / p.pk_per_sample) : 1.f;
            fast_model8<NE>(p, fx, fec, feu, clamp, s_thr, fT);
          } else {
            float thr8[8];
            if (clamp && p.pk_per_sample != 0) {
              const float tpk = __ldg(p.thr + (uint32_t)(pk / p.pk_per_sample));
#pragma unroll
              for (int i = 0; i < 8; ++i) thr8[i] = tpk;
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i) thr8[i] = clamp ? __ldg(p.thr + (e + i) / p.per_sample) : 1.f;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) fT[i] = model_value<NE>(p, fx[i], fec[i], NE == 2 ? feu[i] : 0.f, thr8[i], clamp);
          }
          Raw<TS> rmo;
          round_pack(rmo, fT);
          if (gmo != nullptr) stg_pk(gmo + e, rmo);
        } else {
          unpack(rm0[u], fT);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) fo[i] = unipc_value<TS>(up, fx[i], fT[i], fm1[i], fm2[i], fm3[i], fc[i]);
        if (goc != nullptr) {
          Raw<TS> rc;
          pack(rc, fc);
          stg_pk(goc + e, rc);
        }
        if (up.pp > 0) {
          Raw<TS> ro;
          pack(ro, fo);
          stg_pk(go + e, ro);
          if (go2 != nullptr) stg_pk(go2 + e, ro);
        }
      }
    }
  }
}

// generic element-wise variant: any dtype pair, any alignment, tails
__global__ void __launch_bounds__(256) k_step_unipc_scalar(const __grid_constant__ UniParams up) {
  const KParams& p = up.k;
  const int sd = p.state_dtype, md = p.model_dtype;
  const UniReads rd = uni_reads(up.pc, up.pp);
  const bool clamp = p.n_model > 0 && p.thr != nullptr;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (size_t)gridDim.x * blockDim.x) {
    const float x = load_any(p.x, sd, i);
    const float m1 = rd.m1 ? load_any(p.m1, sd, i) : 0.f;
    const float m2 = rd.m2 ? load_any(p.m2, sd, i) : 0.f;
    const float m3 = rd.m3 ? load_any(up.m3, sd, i) : 0.f;
    float T;
    if (p.n_model > 0) {
      const float ec = load_any(p.ec, md, i);
      const float eu = p.n_model == 2 ? load_any(p.eu, md, i) : 0.f;
      const float thr = clamp ? p.thr[(i + p.elem_offset) / p.per_sample] : 1.f;
      const float mv = p.n_model == 2 ? model_value<2>(p, x, ec, eu, thr, clamp) : model_value<1>(p, x, ec, eu, thr, clamp);
      T = round_any(sd, mv);
      if (p.m_out) store_any(p.m_out, sd, i, mv);
    } else {
      T = load_any(p.m0, sd, i);
    }
    float xc, o;
    switch (sd) {
      case DPM_BF16: o = unipc_value<__nv_bfloat16>(up, x, T, m1, m2, m3, xc); break;
      case DPM_F16: o = unipc_value<__half>(up, x, T, m1, m2, m3, xc); break;
      default: o = unipc_value<float>(up, x, T, m1, m2, m3, xc); break;
    }
    if (up.out_c) store_any(up.out_c, sd, i, xc);
    if (up.pp > 0) {
      store_any(p.out, sd, i, o);
      if (p.out2) store_any(p.out2, sd, i, o);
    }
  }
}

typedef void (*UniKernel)(const UniParams);

int launch_step_unipc(const UniParams& up, const Tuning& t, cudaStream_t stream) {
  const KParams& p = up.k;
  const bool fast = fast_path_ok(p);
  const int md = p.n_model == 0 ? p.state_dtype : p.model_dtype;
  UniKernel k = with_packet_pair(md, p.state_dtype, [&](auto pair) -> UniKernel {
    using TE = typename decltype(pair)::TE;
    using TS = typename decltype(pair)::TS;
    switch (p.n_model) {
      case 0:
        if constexpr (std::is_same_v<TE, TS>) return k_step_unipc<TE, TS, 0, true>;
        return nullptr;
      case 1: return fast ? k_step_unipc<TE, TS, 1, true> : k_step_unipc<TE, TS, 1, false>;
      case 2: return fast ? k_step_unipc<TE, TS, 2, true> : k_step_unipc<TE, TS, 2, false>;
    }
    return nullptr;
  });
  if (k == nullptr) return 1;  // other dtype pairs: the generic kernel
  const int threads = t.threads > 0 && t.threads <= kUniThreads ? t.threads : kUniThreads;
  const uint64_t tile_pk = (uint64_t)threads * kUniUnroll;
  const uint64_t tiles = ((uint64_t)p.npk + tile_pk - 1) / tile_pk;
  const uint64_t cap = t.ctas_per_sm > 0 ? (uint64_t)sm_count() * t.ctas_per_sm : tiles;
  const uint32_t grid = (uint32_t)(tiles < cap ? tiles : cap);
  if (grid == 0) return 0;
  cudaError_t le = launch_pdl(k, grid, (unsigned)threads, 0, stream, up);
  if (le != cudaSuccess) return launch_error("UniPC step launch failed", le);
  count_launch();
  return 0;
}

int launch_step_unipc_scalar(const UniParams& up, cudaStream_t stream) {
  if (up.k.n == 0) return 0;
  const int threads = 256;
  const uint64_t blocks = (up.k.n + threads - 1) / threads;
  const uint64_t cap = (uint64_t)sm_count() * 8;
  const uint32_t grid = (uint32_t)(blocks < cap ? blocks : cap);
  k_step_unipc_scalar<<<grid, threads, 0, stream>>>(up);
  count_launch();
  return 0;
}

}  // namespace dpm
