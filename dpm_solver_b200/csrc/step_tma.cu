// step_tma.cu -- variant 1: TMA bulk staging through a shared-memory ring (fast path only: noise-parameterised
// networks, exact constant division -- common.cuh fast_model8 / fast_update8).
//
// Persistent CTAs. One elected thread moves whole tiles with 1-D bulk async copies
// (cp.async.bulk, SASS UBLKCP): global -> shared completes on an mbarrier (complete_tx),
// shared -> global is a bulk store tracked by bulk groups. The other threads only touch
// shared memory (LDS.128 / STS.128) and registers. kStages tiles are in flight per CTA, so
// the bytes in flight per SM are decoupled from register count and occupancy.
//
// Ring protocol for tile i of a CTA (stage s = i % S):
//   wait full[s] (parity (i/S)&1) -> compute, write results into out-buffers of stage s ->
//   fence.proxy.async -> thread 0: bulk wait_group.read(S-2) (frees the out-buffers of the
//   next stage) -> __syncthreads -> thread 0: bulk-store stage s, commit, then refill the
//   input buffers of stage s with tile i+S.
#include "common.cuh"
#include "launch.cuh"

namespace dpm {

// packets per thread per tile (tile = threads * kUnits packets), compile time: both packets' LDS issue before the
// first use
constexpr int kUnits = 2;
constexpr int kTmaMaxThreads = 512;
constexpr int kMaxStages = 8;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read(int pending) {
  switch (pending) {
    case 0: asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); break;
    case 1: asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); break;
    case 2: asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory"); break;
    case 3: asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory"); break;
    case 4: asm volatile("cp.async.bulk.wait_group.read 4;" ::: "memory"); break;
    case 5: asm volatile("cp.async.bulk.wait_group.read 5;" ::: "memory"); break;
    default: asm volatile("cp.async.bulk.wait_group.read 6;" ::: "memory"); break;
  }
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// byte offsets of the per-stream tile buffers inside one stage
struct StageLayout {
  uint32_t x, xe, ec, eu, m0, m1, m2, mo, o;  // 0xffffffff = stream absent
  uint32_t bytes;                          // stage size
};

// shared-memory packet access by 32-bit shared-window address (no generic-pointer arithmetic in the loop)
__device__ __forceinline__ void lds_pk32(Raw<float>& v, uint32_t a) {
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.r[0]), "=r"(v.r[1]), "=r"(v.r[2]), "=r"(v.r[3]) : "r"(a));
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4+16];" : "=r"(v.r[4]), "=r"(v.r[5]), "=r"(v.r[6]), "=r"(v.r[7]) : "r"(a));
}
template <typename T16>
__device__ __forceinline__ void lds_pk32(Raw<T16>& v, uint32_t a) {
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.r[0]), "=r"(v.r[1]), "=r"(v.r[2]), "=r"(v.r[3]) : "r"(a));
}
__device__ __forceinline__ void sts_pk32(uint32_t a, const Raw<float>& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(v.r[0]), "r"(v.r[1]), "r"(v.r[2]), "r"(v.r[3]) : "memory");
  asm volatile("st.shared.v4.b32 [%0+16], {%1,%2,%3,%4};" ::"r"(a), "r"(v.r[4]), "r"(v.r[5]), "r"(v.r[6]), "r"(v.r[7]) : "memory");
}
template <typename T16>
__device__ __forceinline__ void sts_pk32(uint32_t a, const Raw<T16>& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(v.r[0]), "r"(v.r[1]), "r"(v.r[2]), "r"(v.r[3]) : "memory");
}
__device__ __forceinline__ void bulk_g2s32(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void bulk_s2g32(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx32(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait32(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}

// Fast path only (launch_step_tma: fast_path_ok and no per-sample threshold): noise-parameterised network,
// exact constant division. Everything that is uniform over a tile lives in uniform registers, computed once per
// tile from 32-bit quantities (npk < 2^32): shared-window addresses of the stage's stream buffers, the tile's
// packet count, the ring slot and its parity (counters, no division).
template <typename TE, typename TS, int NE, int FORM>
__global__ void __launch_bounds__(kTmaMaxThreads)
    k_step_tma(const __grid_constant__ KParams p, const __grid_constant__ StageLayout L,
               const int stages, const int /*units: compile time (kUnits)*/) {
  constexpr bool kX = form_reads(FORM).x, kM1 = form_reads(FORM).m1, kM2 = form_reads(FORM).m2;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t sbar = smem_u32(smem);           // [kMaxStages] mbarriers
  const uint32_t sring = sbar + 128;

  const uint32_t tid = threadIdx.x;
  const uint32_t nthr = blockDim.x;
  const uint32_t tile_pk = nthr * kUnits;
  // Tiles go round-robin over the persistent grid: at any moment all CTAs read neighbouring addresses of each
  // stream (one sequential sweep per tensor). Giving every CTA its own contiguous range removes the whole-tile
  // quantisation of the grid but scatters (CTAs x streams) concurrent streams over HBM and measured slower on the
  // first target GPU: kept round-robin.
  const uint32_t ntiles = (p.npk + tile_pk - 1) / tile_pk;
  const bool has_x = kX || (NE > 0 && p.use_xe);  // state slot: x, or xe when no update
  const bool sep_xe = (NE > 0) && p.use_xe && kX && !p.xe_is_x;  // extra slot: evaluation state
  const bool has_mo = (NE > 0) && (p.m_out != nullptr);
  const bool has_o2 = (FORM != DPM_FORM_NONE) && (p.out2 != nullptr);
  const char* gstate = static_cast<const char*>(kX ? p.x : p.xe);
  constexpr uint32_t kBS = Traits<TS>::kBytes * kPacket, kBM = Traits<TE>::kBytes * kPacket;   // bytes per packet

  pdl_trigger();
  if (tid == 0) {
    for (int s = 0; s < stages; ++s) mbar_init(reinterpret_cast<uint64_t*>(smem) + s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();   // everything above overlapped the previous launch's tail; global memory from here on

  auto issue_loads = [&](uint32_t tile, uint32_t s) {
    const uint32_t pk0 = tile * tile_pk;
    const uint32_t pk = min(p.npk - pk0, tile_pk);
    const uint32_t bs = pk * kBS, bm = pk * kBM;
    const uint64_t os = (uint64_t)pk0 * kBS, om = (uint64_t)pk0 * kBM;
    const uint32_t st = sring + s * L.bytes, bar = sbar + s * 8;
    uint32_t tx = 0;
    if (has_x) tx += bs;
    if (sep_xe) tx += bs;
    if (NE >= 1) tx += bm;
    if (NE == 2) tx += bm;
    if (NE == 0) tx += bs;
    if (kM1) tx += bs;
    if (kM2) tx += bs;
    mbar_expect_tx32(bar, tx);
    if (has_x) bulk_g2s32(st + L.x, gstate + os, bs, bar);
    if (sep_xe) bulk_g2s32(st + L.xe, static_cast<const char*>(p.xe) + os, bs, bar);
    if (NE >= 1) bulk_g2s32(st + L.ec, static_cast<const char*>(p.ec) + om, bm, bar);
    if (NE == 2) bulk_g2s32(st + L.eu, static_cast<const char*>(p.eu) + om, bm, bar);
    if (NE == 0) bulk_g2s32(st + L.m0, static_cast<const char*>(p.m0) + os, bs, bar);
    if (kM1) bulk_g2s32(st + L.m1, static_cast<const char*>(p.m1) + os, bs, bar);
    if (kM2) bulk_g2s32(st + L.m2, static_cast<const char*>(p.m2) + os, bs, bar);
  };

  if (tid == 0) {
    for (int s = 0; s < stages; ++s) {
      const uint32_t tile = blockIdx.x + (uint32_t)s * gridDim.x;
      if (tile < ntiles) issue_loads(tile, (uint32_t)s);
    }
  }

  uint32_t slot = 0, parity = 0;
  for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const uint32_t st = sring + slot * L.bytes;
    const uint32_t pk0 = tile * tile_pk;
    const uint32_t pk_here = min(p.npk - pk0, tile_pk);

    mbar_wait32(sbar + slot * 8, parity);

    // ---- load both packets of this thread, then compute ----
    Raw<TS> rx[kUnits], rxe[kUnits], rm0[kUnits], rm1[kUnits], rm2[kUnits];
    Raw<TE> rec[kUnits], reu[kUnits];
#pragma unroll
    for (int u = 0; u < kUnits; ++u) {
      const uint32_t lp = u * nthr + tid;  // packet inside the tile
      if (lp < pk_here) {
        if (has_x) lds_pk32(rx[u], st + L.x + lp * kBS);
        if (sep_xe) lds_pk32(rxe[u], st + L.xe + lp * kBS);
        if (kM1) lds_pk32(rm1[u], st + L.m1 + lp * kBS);
        if (kM2) lds_pk32(rm2[u], st + L.m2 + lp * kBS);
        if (NE >= 1) lds_pk32(rec[u], st + L.ec + lp * kBM);
        if (NE == 2) lds_pk32(reu[u], st + L.eu + lp * kBM);
        if (NE == 0) lds_pk32(rm0[u], st + L.m0 + lp * kBS);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnits; ++u) {
      const uint32_t lp = u * nthr + tid;
      if (lp < pk_here) {
        float fx[8], fT[8], fm1[8], fm2[8], fo[8];
        if (has_x) unpack(rx[u], fx);
        if (kM1) unpack(rm1[u], fm1);
        if (kM2) unpack(rm2[u], fm2);
        if (NE > 0) {
          float fec[8], feu[8];
          unpack(rec[u], fec);
          if (NE == 2) unpack(reu[u], feu);
          if (sep_xe) {
            float fxe[8];
            unpack(rxe[u], fxe);
            fast_model8<NE>(p, fxe, fec, feu, false, 1.f, fT);
          } else {
            fast_model8<NE>(p, fx, fec, feu, false, 1.f, fT);   // fx is only read when the conversion needs it (then has_x)
          }
          Raw<TS> rmo;
          round_pack(rmo, fT);
          if (has_mo) sts_pk32(st + L.mo + lp * kBS, rmo);
        } else {
          unpack(rm0[u], fT);
        }
        if (FORM != DPM_FORM_NONE) {
          fast_update8<FORM>(p, fx, fT, fm1, fm2, fo);
          Raw<TS> r;
          pack(r, fo);
          sts_pk32(st + L.o + lp * kBS, r);
        }
      }
    }
    fence_async_smem();  // generic-proxy writes -> visible to the async proxy (bulk store)
    if (tid == 0) bulk_wait_read(stages - 2);
    __syncthreads();
    if (tid == 0) {
      const uint32_t bs = pk_here * kBS;
      const uint64_t os = (uint64_t)pk0 * kBS;
      if (has_mo) bulk_s2g32(static_cast<char*>(p.m_out) + os, st + L.mo, bs);
      if (FORM != DPM_FORM_NONE) {
        bulk_s2g32(static_cast<char*>(p.out) + os, st + L.o, bs);
        if (has_o2) bulk_s2g32(static_cast<char*>(p.out2) + os, st + L.o, bs);
      }
      bulk_commit();
      const uint32_t next = tile + (uint32_t)stages * gridDim.x;     // < 2^32: ntiles * (1 + stages) never gets near it
      if (next < ntiles && next > tile) issue_loads(next, slot);
    }
    if (++slot == (uint32_t)stages) { slot = 0; parity ^= 1u; }
  }
  if (tid == 0) bulk_wait_all();
}

typedef void (*TmaKernel)(const KParams, const StageLayout, const int, const int);

int launch_step_tma(const KParams& p, const Tuning& t, cudaStream_t stream) {
  if (!fast_path_ok(p) || p.thr != nullptr) return 1;   // other parameterisations, non-refinable divisors, per-sample
                                                        // thresholds: the direct variant
  TmaKernel k = pick_step<TmaKernel>(p, [](auto pair, auto ne, auto form) -> TmaKernel {
    using Pair = decltype(pair);
    return k_step_tma<typename Pair::TE, typename Pair::TS, decltype(ne)::value, decltype(form)::value>;
  });
  if (k == nullptr) return 1;
  const FormReads reads = form_reads(p.form);
  const bool need_x = reads.x;
  const uint32_t ss = p.state_dtype == DPM_F32 ? 4 : 2, ms = p.model_dtype == DPM_F32 ? 4 : 2;
  const bool has_x = need_x || (p.n_model > 0 && p.use_xe);   // state slot: x, or xe when no update
  const bool sep_xe = p.n_model > 0 && p.use_xe && need_x && !p.xe_is_x;
  const bool has_mo = p.n_model > 0 && p.m_out != nullptr;
  // the shared-memory streams of a stage, one per take() below
  const int n_streams = has_x + sep_xe + p.n_model + (p.n_model == 0) + reads.m1 + reads.m2 + has_mo + need_x;
  // Launch shape, decided inside the sampling loop on the first target GPU (not re-swept on H100): launches
  // with <= 4 shared-memory streams run best as 256 threads x 3 CTAs/SM, 5 streams as 256 x 2; when the tile is
  // also stored twice (out2: 6 HBM streams, the CFG steps of c3) one 512-thread CTA per SM with two 80 KB stages.
  int def_threads = 256, def_ctas = 2;
  const int hbm_streams = n_streams + (need_x && p.out2 != nullptr);
  if (ss == 2 && ms == 2 && n_streams <= 4) def_ctas = 3;
  else if (ss == 2 && ms == 2 && hbm_streams >= 6) { def_threads = 512; def_ctas = 1; }
  const int ctas = t.ctas_per_sm > 0 ? t.ctas_per_sm : def_ctas;
  // smem budget per CTA: the SM's 228 KB (H100) hold `ctas` CTAs (1 KB reserved per CTA)
  const size_t per_cta = (size_t)(228 * 1024) / ctas - 1024;
  const size_t budget = per_cta < (size_t)max_smem_optin() ? per_cta : (size_t)max_smem_optin();

  StageLayout L;
  int threads = 0, stages = 0;
  const int units = kUnits;   // compile-time constant of the kernel
  // tile = threads * units packets. Default 256 threads x 2 CTAs/SM (512 resident threads):
  // sweeps showed two stages at that size beat more, smaller stages; the tile only
  // shrinks when two stages of it do not fit.
  const int cand[4] = {t.threads > 0 ? t.threads : def_threads, t.threads > 0 || def_threads > 256 ? 256 : 128, 64, 32};
  for (int c = 0; c < (t.threads > 0 ? 1 : 4); ++c) {
    const uint32_t tile_el = (uint32_t)cand[c] * units * kPacket;
    uint32_t o = 0;
    auto take = [&](bool on, uint32_t es) { uint32_t r = 0xffffffffu; if (on) { r = o; o += tile_el * es; } return r; };
    L.x = take(has_x, ss);
    L.xe = take(sep_xe, ss);
    L.ec = take(p.n_model >= 1, ms);
    L.eu = take(p.n_model == 2, ms);
    L.m0 = take(p.n_model == 0, ss);
    L.m1 = take(reads.m1, ss);
    L.m2 = take(reads.m2, ss);
    L.mo = take(has_mo, ss);
    L.o = take(need_x, ss);
    L.bytes = o;
    int st = (int)((budget - 128) / L.bytes);
    if (st > kMaxStages) st = kMaxStages;
    threads = cand[c];
    stages = st;
    if (st >= 2) break;
  }
  if (stages < 2) return 1;
  const size_t smem = 128 + (size_t)stages * L.bytes;

  const uint32_t tile_pk = (uint32_t)threads * units;
  const uint64_t ntiles = ((uint64_t)p.npk + tile_pk - 1) / tile_pk;
  const uint64_t cap = (uint64_t)sm_count() * ctas;
  const uint32_t grid = (uint32_t)(ntiles < cap ? ntiles : cap);
  if (grid == 0) return 0;
  int rc = ensure_max_smem(reinterpret_cast<const void*>(k));  // once per kernel and device
  if (rc != 0) return rc;
  cudaError_t le = launch_pdl(k, grid, (unsigned)threads, smem, stream, p, L, stages, units);
  if (le != cudaSuccess) return launch_error("TMA step launch failed", le);
  count_launch();
  return 0;
}

// ---- cat([x] * 2): one read, two writes, no register traffic -----------------------------------------
// model_wrapper.model_fn builds the network's doubled CFG batch with torch.cat([x] * 2) (:326). Inside the
// sampling loop the update kernel writes x_t into both halves itself (out2); this kernel serves the first
// evaluation of a run: each tile is bulk-loaded into shared memory once and bulk-stored twice.
constexpr int kDupStages = 4;
constexpr uint32_t kDupTileBytes = 32 * 1024;

__global__ void __launch_bounds__(32) k_dup_tma(const char* __restrict__ src, char* __restrict__ dst0,
                                                char* __restrict__ dst1, const uint64_t bytes) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t full = smem_u32(smem);   // [kDupStages] mbarriers
  const uint32_t ring = full + 128;
  const uint64_t ntiles = (bytes + kDupTileBytes - 1) / kDupTileBytes;
  if (threadIdx.x != 0) return;     // one elected thread drives the copy engine; the warp exists for the launch only
  for (int s = 0; s < kDupStages; ++s) mbar_init(reinterpret_cast<uint64_t*>(smem) + s, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  auto load = [&](uint64_t tile, int s) {
    const uint64_t b0 = tile * kDupTileBytes;
    const uint32_t nb = (uint32_t)((bytes - b0) < kDupTileBytes ? (bytes - b0) : kDupTileBytes);
    mbar_expect_tx32(full + s * 8, nb);
    bulk_g2s32(ring + s * kDupTileBytes, src + b0, nb, full + s * 8);
  };
  for (int s = 0; s < kDupStages; ++s) {
    const uint64_t tile = (uint64_t)blockIdx.x + (uint64_t)s * gridDim.x;
    if (tile < ntiles) load(tile, s);
  }
  uint32_t it = 0;
  for (uint64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const int s = it % kDupStages;
    mbar_wait32(full + s * 8, (it / kDupStages) & 1u);
    const uint64_t b0 = tile * kDupTileBytes;
    const uint32_t nb = (uint32_t)((bytes - b0) < kDupTileBytes ? (bytes - b0) : kDupTileBytes);
    bulk_s2g32(dst0 + b0, ring + s * kDupTileBytes, nb);
    bulk_s2g32(dst1 + b0, ring + s * kDupTileBytes, nb);
    bulk_commit();
    const uint64_t next = tile + (uint64_t)kDupStages * gridDim.x;
    if (next < ntiles) {
      bulk_wait_read(0);            // the stores have read the stage: it may be refilled
      load(next, s);
    }
  }
  bulk_wait_all();
}

// returns 0 on launch, 1 when the request is not served here (unaligned / tiny: caller falls back to copies)
int launch_duplicate(void* dst, const void* src, uint64_t bytes, cudaStream_t stream) {
  if (bytes == 0) return 0;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (!al16(dst) || !al16(src) || (bytes & 15) != 0) return 1;
  const uint64_t ntiles = (bytes + kDupTileBytes - 1) / kDupTileBytes;
  const uint64_t cap = (uint64_t)sm_count() * 1;     // 128 KB of ring per CTA: one CTA per SM keeps 128 KB in flight
  const uint32_t grid = (uint32_t)(ntiles < cap ? ntiles : cap);
  const size_t smem = 128 + (size_t)kDupStages * kDupTileBytes;
  int rc = ensure_max_smem(reinterpret_cast<const void*>(k_dup_tma));
  if (rc != 0) return rc;
  k_dup_tma<<<grid, 32, smem, stream>>>(static_cast<const char*>(src), static_cast<char*>(dst),
                                        static_cast<char*>(dst) + bytes, bytes);
  count_launch();
  return 0;
}

}  // namespace dpm
