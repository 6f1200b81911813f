// words.cu -- the per-sample guidance words: fp64 reductions over the network outputs that run before the fused step.
// Every pass is one skeleton with a compile-time policy: CTA (b, c) reduces chunk c of sample b to the pass's fp64
// partials (k_words_partial), then one thread per sample merges its chunks in chunk order and writes the words (the
// pass's final kernel). Thread tid owns chunk elements (u*256 + tid)*8 + i, u = 0..3, i = 0..7, on the vector and the
// element-wise path alike, and every sum runs in a fixed order, so the words of sample b depend on its values only --
// not on the batch, the sample's position or the alignment. Two launches, no allocation, no sync.
// (This file builds with -fmad=false: no product below is contracted into an fma.)
#include <initializer_list>
#include <tuple>
#include <type_traits>
#include <utility>

#include "common.cuh"
#include "launch.cuh"

namespace dpm {

constexpr int kWThreads = 256;
constexpr int kWChunk = 8192;                          // elements per CTA
constexpr int kWU = kWChunk / kPacket / kWThreads;     // packets per thread: 4

// The leading member of every pass's parameters.
struct WordsGeom {
  double* partial;       // [n_samples * chunks][the pass's sums]
  uint64_t per_sample;
  uint64_t n_samples;
  uint32_t chunks;       // per sample
};

static uint64_t words_chunks(uint64_t per_sample) { return (per_sample + kWChunk - 1) / kWChunk; }

size_t words_workspace_bytes(uint64_t n_samples, uint64_t per_sample, int sums) {
  if (per_sample == 0 || n_samples == 0) return 0;
  return (size_t)(n_samples * words_chunks(per_sample)) * sums * sizeof(double);
}

// The chunk of this CTA: its sample, its live element count and its first element.
struct Chunk {
  uint64_t sample;
  uint32_t cnt;
  size_t e0;
};
__device__ __forceinline__ Chunk chunk_of(const WordsGeom& g) {
  const uint64_t sample = blockIdx.x / g.chunks;
  const uint64_t c_begin = (uint64_t)(blockIdx.x % g.chunks) * kWChunk;
  const uint64_t c_end = c_begin + kWChunk < g.per_sample ? c_begin + kWChunk : g.per_sample;
  return {sample, (uint32_t)(c_end - c_begin), sample * g.per_sample + c_begin};
}

// deterministic CTA sum of one double per thread (butterfly within the warps, then the warps in order)
__device__ __forceinline__ double cta_sum(double v, double* warp_part) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();   // warp_part may still be read from the previous call
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < kWThreads / 32; ++w) s += warp_part[w];
  return s;
}

// One input stream of a pass: T is its element type on the vector path, dtype its storage on the element-wise path.
// Opt: the pointer may be NULL, and the stream then reads as 0 (load_packet leaves it unset, visit selects the 0).
template <typename T, bool Opt = false>
struct In {
  using Elem = T;
  static constexpr bool kOpt = Opt;
  const void* p;
  int dtype;
  __device__ __forceinline__ bool read() const { return !Opt || p != nullptr; }
};
template <typename T, bool Opt>
__device__ __forceinline__ void load_packet(const In<T, Opt>& s, size_t e, float (&f)[8]) {
  Raw<T> r;
  if (s.read()) ldg_pk(r, static_cast<const T*>(s.p) + e);
  if (s.read()) unpack(r, f);
}
template <typename T, bool Opt>
__device__ __forceinline__ float load_one(const In<T, Opt>& s, size_t e) {
  return Opt && s.p == nullptr ? 0.f : load_any(s.p, s.dtype, e);
}

// Calls f(u, i, v) for each live element (u, i) of this thread, v[k] the element's value in stream k, in the order
// u = 0..3, i = 0..7. VEC: per_sample % 8 == 0 and every stream aligned (whole packets, ldg_pk), else load_any. When f
// returns a float, it is written to `out` (NULL: not written) at the element, as one packet on the vector path.
// Ahead (vector path, streams of one type, no output): every packet of the thread is loaded before the first call of
// f, so all kWU*N loads are in flight at once. For a pass that holds its whole chunk in registers, and so runs one CTA
// per SM, these loads are its only memory-level parallelism; the other passes load and reduce packet by packet.
template <bool VEC, bool Ahead = false, typename F, typename... S>
__device__ __forceinline__ void visit(const Chunk& c, float* out, F&& f, const S&... s) {
  constexpr int N = sizeof...(S);
  constexpr bool kOut = !std::is_void_v<decltype(f(0, 0, std::declval<const float (&)[N]>()))>;
  if constexpr (VEC && Ahead) {
    using T = typename std::tuple_element_t<0, std::tuple<S...>>::Elem;
    static_assert(!kOut && ((std::is_same_v<typename S::Elem, T> && !S::kOpt) && ...), "one type, no output");
    const void* const ptr[N] = {s.p...};
    Raw<T> raw[N][kWU];
#pragma unroll
    for (int u = 0; u < kWU; ++u) {
      const uint32_t pk = u * kWThreads + threadIdx.x;
      if (pk * kPacket < c.cnt) {
#pragma unroll
        for (int j = 0; j < N; ++j) ldg_pk(raw[j][u], static_cast<const T*>(ptr[j]) + c.e0 + (size_t)pk * kPacket);
      }
    }
#pragma unroll
    for (int u = 0; u < kWU; ++u) {
      const uint32_t pk = u * kWThreads + threadIdx.x;
      if (pk * kPacket < c.cnt) {
        float v[N][8];
#pragma unroll
        for (int j = 0; j < N; ++j) unpack(raw[j][u], v[j]);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float x[N];
#pragma unroll
          for (int j = 0; j < N; ++j) x[j] = v[j][i];
          f(u, i, x);
        }
      }
    }
    return;
  }
#pragma unroll
  for (int u = 0; u < kWU; ++u) {
    const uint32_t pk = u * kWThreads + threadIdx.x;
    if (VEC) {
      if (pk * kPacket < c.cnt) {
        const size_t e = c.e0 + (size_t)pk * kPacket;
        float v[N][8];
        const bool rd[N] = {s.read()...};   // a stream that is not read gives 0, selected per element at its use
        int k = 0;
        (load_packet(s, e, v[k++]), ...);
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float x[N];
#pragma unroll
          for (int j = 0; j < N; ++j) x[j] = rd[j] ? v[j][i] : 0.f;
          if constexpr (kOut) o[i] = f(u, i, x);
          else f(u, i, x);
        }
        if constexpr (kOut) {
          if (out != nullptr) {
            Raw<float> r;
            pack(r, o);
            stg_pk(out + e, r);
          }
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t j = pk * kPacket + i;
        if (j < c.cnt) {
          const size_t e = c.e0 + j;
          float x[N];
          int k = 0;
          ((x[k++] = load_one(s, e)), ...);
          if constexpr (kOut) {
            const float r = f(u, i, x);
            if (out != nullptr) out[e] = r;
          } else {
            f(u, i, x);
          }
        }
      }
    }
  }
}

// The partials of one chunk: Pass::sums fills the CTA's kSums fp64 values, thread 0 stores them.
template <class Pass, typename TE, typename TS, bool VEC>
__global__ void __launch_bounds__(kWThreads) k_words_partial(const __grid_constant__ typename Pass::Params p) {
  __shared__ double warp_part[kWThreads / 32];
  double s[Pass::kSums];
  Pass::template sums<TE, TS, VEC>(p, chunk_of(p.g), warp_part, s);
  if (threadIdx.x == 0) {
    double* o = p.g.partial + (size_t)blockIdx.x * Pass::kSums;
#pragma unroll
    for (int k = 0; k < Pass::kSums; ++k) o[k] = s[k];
  }
}

// The first NS of the ns partials per chunk of sample b, each merged from 0.0 in chunk order.
template <int NS>
__device__ __forceinline__ void merge_sums(const WordsGeom& g, uint64_t b, int ns, double (&s)[NS]) {
  const double* part = g.partial + b * g.chunks * ns;
#pragma unroll
  for (int k = 0; k < NS; ++k) s[k] = 0.0;
  for (uint32_t c = 0; c < g.chunks; ++c) {
#pragma unroll
    for (int k = 0; k < NS; ++k)
      if (k < ns) s[k] += part[c * ns + k];
  }
}

static inline bool packet_aligned(const void* q, int dtype) {
  return (reinterpret_cast<uintptr_t>(q) & (dtype == DPM_F32 ? 31 : 15)) == 0;
}

// The host side every pass shares: the workspace and chunk-count checks, the vector decision (per_sample whole packets
// and every stream aligned; a NULL stream is not read), the dtype dispatch (the packet pair (md, sd) on the vector path,
// <float, float, false> element-wise for any dtype, alignment or sample size), the two launches and their count.
template <class Pass>
static int launch_words(const char* what, typename Pass::Params& p, void (*final)(typename Pass::Params), int md,
                        int sd, std::initializer_list<std::pair<const void*, int>> streams, void* ws, size_t ws_bytes,
                        cudaStream_t stream) {
  p.g.chunks = (uint32_t)words_chunks(p.g.per_sample);
  p.g.partial = static_cast<double*>(ws);
  if (ws == nullptr || ws_bytes < words_workspace_bytes(p.g.n_samples, p.g.per_sample, Pass::kWorkspaceSums) ||
      (reinterpret_cast<uintptr_t>(ws) & 7)) {
    set_error("%s: workspace too small or not 8-byte aligned", what);
    return DPM_ERR_ARG;
  }
  if (p.g.n_samples * p.g.chunks > 0x7fffffffull) { set_error("%s: too many chunks", what); return DPM_ERR_UNSUPPORTED; }
  bool vec = p.g.per_sample % kPacket == 0;
  for (const auto& s : streams) vec = vec && (s.first == nullptr || packet_aligned(s.first, s.second));
  typedef void (*PKernel)(const typename Pass::Params);
  PKernel k = nullptr;
  if (vec) {
    k = with_packet_pair(md, sd, [&](auto pair) -> PKernel {
      using Pair = decltype(pair);
      if constexpr (Pass::kState || std::is_same_v<typename Pair::TE, typename Pair::TS>)
        return k_words_partial<Pass, typename Pair::TE, typename Pair::TS, true>;
      return nullptr;
    });
  }
  if (k == nullptr) k = k_words_partial<Pass, float, float, false>;
  k<<<(unsigned)(p.g.n_samples * p.g.chunks), kWThreads, 0, stream>>>(p);
  final<<<(unsigned)((p.g.n_samples + kWThreads - 1) / kWThreads), kWThreads, 0, stream>>>(p);
  count_launch();
  count_launch();
  return DPM_OK;
}

// ---- guidance rescale ratio (dpm_cfg_rescale_ratio) ------------------------------------------------------------------
//   g = out_u + s*(out_c - out_u)   (the step kernels' combine, :330)
//   r[b] = fl32(std(out_c[b])) / fl32(std(g[b])),  std unbiased, in fp64
// CTA (b, c) holds chunk c of sample b in registers, takes its fp64 mean (first reduction) and the sum of squared
// deviations from that mean (second reduction, exact for any mean/std ratio an fp32 sample can have); the final kernel
// merges the chunks of a sample in chunk order (Chan et al.'s pairwise update).
struct RParams {
  WordsGeom g;           // partial: [n_samples * chunks][4]: mean_c, M2_c, mean_g, M2_g
  const void* ec;
  const void* eu;
  float* ratio;          // [n_samples]
  int32_t dtype;
  float guidance;
  const float* gscale;   // per-sample scales [n_samples] in place of `guidance` (<PG = true> only)
};

// PG: per-sample guidance (dpm_cfg_rescale_ratio_guided): g = out_u + s_b*(out_c - out_u) with the sample's scale
template <bool PG>
struct RatioPass {
  using Params = RParams;
  static constexpr int kSums = 4, kWorkspaceSums = 4;
  static constexpr bool kState = false;
  template <typename TE, typename TS, bool VEC>
  __device__ static void sums(const Params& p, const Chunk& c, double* warp_part, double (&s)[kSums]) {
    float s_b;
    if constexpr (PG) s_b = __ldg(p.gscale + c.sample);
    else s_b = p.guidance;
    float fc[kWU][8], fg[kWU][8];
    // The chunk stays in registers (one CTA per SM). fp32 packets are all loaded ahead; 16-bit ones load faster
    // packet by packet (measured on H100: bf16 [4096,4,64,64] 251 us against 273 us loaded ahead).
    visit<VEC, std::is_same_v<TE, float>>(c, nullptr, [&](int u, int i, const float (&v)[2]) {
      fc[u][i] = v[0];
      fg[u][i] = v[1] + s_b * (v[0] - v[1]);   // :330
    }, In<TE>{p.ec, p.dtype}, In<TE>{p.eu, p.dtype});
    auto live = [&](int u, int i) { return (uint32_t)((u * kWThreads + threadIdx.x) * kPacket + i) < c.cnt; };
    double sc = 0.0, sg = 0.0;
#pragma unroll
    for (int u = 0; u < kWU; ++u) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (live(u, i)) {
          sc += (double)fc[u][i];
          sg += (double)fg[u][i];
        }
      }
    }
    const double mc = cta_sum(sc, warp_part) / (double)c.cnt;
    const double mg = cta_sum(sg, warp_part) / (double)c.cnt;
    double qc = 0.0, qg = 0.0;
#pragma unroll
    for (int u = 0; u < kWU; ++u) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (live(u, i)) {
          const double dc = (double)fc[u][i] - mc, dg = (double)fg[u][i] - mg;
          qc += dc * dc;
          qg += dg * dg;
        }
      }
    }
    s[0] = mc; s[1] = cta_sum(qc, warp_part); s[2] = mg; s[3] = cta_sum(qg, warp_part);
  }
};

__global__ void __launch_bounds__(kWThreads) k_cfg_ratio_final(const __grid_constant__ RParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kWThreads + threadIdx.x;
  if (b >= p.g.n_samples) return;
  const double* part = p.g.partial + b * p.g.chunks * 4;
  double n = 0.0, mc = 0.0, qc = 0.0, mg = 0.0, qg = 0.0;
  for (uint32_t c = 0; c < p.g.chunks; ++c) {
    const uint64_t c_begin = (uint64_t)c * kWChunk;
    const double nb = (double)((c_begin + kWChunk < p.g.per_sample ? c_begin + kWChunk : p.g.per_sample) - c_begin);
    const double* q = part + (size_t)c * 4;
    if (c == 0) {
      mc = q[0]; qc = q[1]; mg = q[2]; qg = q[3];
    } else {
      const double nab = n + nb, wb = nb / nab, wab = n * nb / nab;
      const double dc = q[0] - mc, dg = q[2] - mg;
      mc = mc + dc * wb;
      qc = (qc + q[1]) + dc * dc * wab;
      mg = mg + dg * wb;
      qg = (qg + q[3]) + dg * dg * wab;
    }
    n += nb;
  }
  // unbiased (torch.std's default correction): one sample gives 0/0 = NaN; each std is rounded to fp32 once
  const float std_c = (float)sqrt(qc / (n - 1.0));
  const float std_g = (float)sqrt(qg / (n - 1.0));
  p.ratio[b] = std_c / std_g;
}

int launch_cfg_rescale_ratio(float* ratio, const void* ec, const void* eu, float guidance, uint64_t per_sample,
                             uint64_t n, int dtype, void* ws, size_t ws_bytes, cudaStream_t stream,
                             const float* gscale) {
  RParams p;
  memset(&p, 0, sizeof(p));
  p.g.per_sample = per_sample; p.g.n_samples = n / per_sample;
  p.ec = ec; p.eu = eu; p.ratio = ratio; p.dtype = dtype; p.guidance = guidance; p.gscale = gscale;
  const auto launch = gscale != nullptr ? launch_words<RatioPass<true>> : launch_words<RatioPass<false>>;
  return launch("cfg rescale", p, k_cfg_ratio_final, dtype, dtype, {{ec, dtype}, {eu, dtype}}, ws, ws_bytes, stream);
}

// ---- APG (dpm_apg_words; Sadat, Hilliges and Weber, "Eliminating Oversaturation and Artifacts of High Guidance
// Scales in Diffusion Models", ICLR 2025) ---------------------------------------------------------------------------
//   c = x0(out_c), u = x0(out_u), D = c - u                       (the step's conversion, each op rounded)
//   R = D, or R = D + beta*R_prev                                  (momentum; written to r_out when set)
//   k = min(1, r/||R||) (r > 0), p = <R, c>/max(||c||, 1e-12)^2
//   A = 1 - (w - 1)*(1 - eta)*k*p,  B = (w - 1)*k                  (fp64, each rounded to fp32 once)
// so that the step's guided prediction c + (w - 1)*(k*R - (1 - eta)*k*p*c) is A*c + B*R. Three sums per chunk.
// Algorithmic bytes per element: x, out_c, out_u read, plus 4 + 4 of R_prev / R with momentum.
struct AParams {
  WordsGeom g;           // partial: [n_samples * chunks][3]: ||R||^2, <R, c>, ||c||^2
  KParams k;             // xe, ec, eu, param, alpha_e, sigma_e (x0 words), guidance, dtypes, dev_coef
  const float* gscale;   // per-sample scales [n_samples], or NULL: k.guidance
  const float* r_prev;   // NULL: R = D
  float* r_out;          // NULL: R is not written
  float* words;          // [2][n_samples]
  float eta, norm_threshold, momentum;
};

struct ApgPass {
  using Params = AParams;
  static constexpr int kSums = 3, kWorkspaceSums = 3;
  static constexpr bool kState = true;   // x is read in the state dtype (TS)
  template <typename TE, typename TS, bool VEC>
  __device__ static void sums(const Params& p, const Chunk& c, double* warp_part, double (&s)[kSums]) {
    KParams k = p.k;
    if (k.dev_coef != nullptr) { k.alpha_e = k.dev_coef[9]; k.sigma_e = k.dev_coef[10]; }
    double srr = 0.0, src = 0.0, scc = 0.0;
    visit<VEC>(c, p.r_out, [&](int, int, const float (&v)[4]) {
      const float xe = v[0], oc = v[1], ou = v[2];   // (named: nvcc then shares one param switch between the two x0)
      const float cc = apg_x0(k, oc, xe);
      const float D = cc - apg_x0(k, ou, xe);
      const float R = p.r_prev != nullptr ? D + p.momentum * v[3] : D;
      srr += (double)R * (double)R;
      src += (double)R * (double)cc;
      scc += (double)cc * (double)cc;
      return R;
    }, In<TS>{k.xe, k.state_dtype}, In<TE>{k.ec, k.model_dtype}, In<TE>{k.eu, k.model_dtype},
       In<float, true>{p.r_prev, DPM_F32});
    s[0] = cta_sum(srr, warp_part);
    s[1] = cta_sum(src, warp_part);
    s[2] = cta_sum(scc, warp_part);
  }
};

__global__ void __launch_bounds__(kWThreads) k_apg_final(const __grid_constant__ AParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kWThreads + threadIdx.x;
  if (b >= p.g.n_samples) return;
  double s[3];
  merge_sums(p.g, b, 3, s);
  const double srr = s[0], src = s[1], scc = s[2];
  double kk = 1.0;
  if (p.norm_threshold > 0.f) {
    const double q = (double)p.norm_threshold / sqrt(srr);
    kk = q < 1.0 ? q : 1.0;
  }
  const double sc = sqrt(scc);
  const double nc = sc < 1e-12 ? 1e-12 : sc;                 // F.normalize's epsilon (a NaN norm stays NaN)
  const double proj = src / (nc * nc);
  const double w = (double)(p.gscale != nullptr ? p.gscale[b] : p.k.guidance);
  const double A = 1.0 - (w - 1.0) * (1.0 - (double)p.eta) * kk * proj;
  const double B = (w - 1.0) * kk;
  p.words[b] = (float)A;
  p.words[p.g.n_samples + b] = (float)B;
}

int launch_apg_words(float* words, const KParams& kp, const float* gscale, float eta, float norm_threshold,
                     float momentum, const float* r_prev, float* r_out, void* ws, size_t ws_bytes, cudaStream_t stream) {
  AParams p;
  memset(&p, 0, sizeof(p));
  p.g.per_sample = kp.per_sample; p.g.n_samples = kp.n / kp.per_sample;
  p.k = kp;
  p.gscale = gscale; p.r_prev = r_prev; p.r_out = r_out; p.words = words;
  p.eta = eta; p.norm_threshold = norm_threshold; p.momentum = momentum;
  return launch_words<ApgPass>("apg words", p, k_apg_final, kp.model_dtype, kp.state_dtype,
                               {{kp.xe, kp.state_dtype}, {kp.ec, kp.model_dtype}, {kp.eu, kp.model_dtype},
                                {r_prev, DPM_F32}, {r_out, DPM_F32}},
                               ws, ws_bytes, stream);
}

// ---- CFG-Zero* (dpm_cfgzero_scale; Fan, Zheng, Yeh and Liu, arXiv:2503.18886) -------------------------------------
// s*_b = fl32(<c_b, u_b> / (||u_b||^2 + 1e-8)) over the two raw network halves of sample b, fp64 sums of the widened
// outputs: no x, no marginals, no dev_coef. Algorithmic bytes: 2*s_model per element.
// ---- TCFG (dpm_tcfg_words; "TCFG: Tangential Damping Classifier-free Guidance", CVPR 2025) -------------------------
// The same pass with three sums, A = ||u||^2, B = <u, c>, C = ||c||^2, and k_tcfg_final in place of k_cfgzero_final:
// the words (wu, wc) of u' = wu*u + wc*c, the projection of u on the first right singular vector of [u; c].
struct ZParams {
  WordsGeom g;           // partial: [n_samples * chunks][NS]: <c, u>, ||u||^2 (CFG-Zero*) or ||u||^2, <u, c>, ||c||^2
  const void* ec;
  const void* eu;
  float* s_out;          // [n_samples] s* (CFG-Zero*) or [n_samples][2] (wu, wc) (TCFG)
  int32_t model_dtype;
};

// NS: the number of sums, 2 (CFG-Zero*) or 3 (TCFG)
template <int NS>
struct PairPass {
  static_assert(NS == 2 || NS == 3, "two or three sums");
  using Params = ZParams;
  static constexpr int kSums = NS, kWorkspaceSums = NS;
  static constexpr bool kState = false;
  template <typename TE, typename TS, bool VEC>
  __device__ static void sums(const Params& p, const Chunk& c, double* warp_part, double (&s)[kSums]) {
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;   // <c, u>, ||u||^2 (NS == 2); ||u||^2, <u, c>, ||c||^2 (NS == 3)
    visit<VEC>(c, nullptr, [&](int, int, const float (&v)[2]) {
      const float cv = v[0], u = v[1];
      if constexpr (NS == 2) {
        s0 += (double)cv * (double)u;
        s1 += (double)u * (double)u;
      } else {
        s0 += (double)u * (double)u;
        s1 += (double)u * (double)cv;
        s2 += (double)cv * (double)cv;
      }
    }, In<TE>{p.ec, p.model_dtype}, In<TE>{p.eu, p.model_dtype});
    s[0] = cta_sum(s0, warp_part);
    s[1] = cta_sum(s1, warp_part);
    if constexpr (NS == 3) s[2] = cta_sum(s2, warp_part);
  }
};

__global__ void __launch_bounds__(kWThreads) k_cfgzero_final(const __grid_constant__ ZParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kWThreads + threadIdx.x;
  if (b >= p.g.n_samples) return;
  double s[2];
  merge_sums(p.g, b, 2, s);
  p.s_out[b] = (float)(s[0] / (s[1] + 1e-8));   // diffusers' cfg_zero_star_scale epsilon
}

// The words of sample b from its merged sums, in fp64 with each op rounded. (p, q) is the top eigenvector of the Gram
// matrix [[A, B], [B, C]], taken from the row without cancellation (h <= 0: row 1, else row 2); with the eigen identity
// the projection <u, v1>*v1 is (p*p*u + p*q*c)/(p*p + q*q). n2 == 0 (A == C and B == 0: no unique top direction, both
// outputs zero included) gives (1, 0), plain CFG; a sum that is not finite gives NaN words.
__global__ void __launch_bounds__(kWThreads) k_tcfg_final(const __grid_constant__ ZParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kWThreads + threadIdx.x;
  if (b >= p.g.n_samples) return;
  double s[3];
  merge_sums(p.g, b, 3, s);
  const double A = s[0], B = s[1], C = s[2];
  float wu, wc;
  if (!(isfinite(A) && isfinite(B) && isfinite(C))) {
    wu = wc = __int_as_float(0x7fffffff);
  } else {
    const double h = 0.5 * (A - C);
    const double r = sqrt(h * h + B * B);
    double pv, qv;
    if (C >= A) { pv = B; qv = (-h) + r; }
    else        { pv = h + r; qv = B; }
    const double pp = pv * pv;
    const double n2 = pp + qv * qv;
    if (n2 == 0.0) { wu = 1.f; wc = 0.f; }
    else { wu = (float)(pp / n2); wc = (float)((pv * qv) / n2); }
  }
  p.s_out[2 * b] = wu;
  p.s_out[2 * b + 1] = wc;
}

template <int NS>
static int launch_pair_pass(void (*final)(ZParams), const char* what, float* s_out, const void* ec, const void* eu,
                            int model_dtype, uint64_t per_sample, uint64_t n, void* ws, size_t ws_bytes,
                            cudaStream_t stream) {
  ZParams p;
  memset(&p, 0, sizeof(p));
  p.g.per_sample = per_sample; p.g.n_samples = n / per_sample;
  p.ec = ec; p.eu = eu; p.s_out = s_out; p.model_dtype = model_dtype;
  return launch_words<PairPass<NS>>(what, p, final, model_dtype, model_dtype, {{ec, model_dtype}, {eu, model_dtype}},
                                    ws, ws_bytes, stream);
}

int launch_cfgzero_scale(float* s_out, const void* ec, const void* eu, int model_dtype, uint64_t per_sample,
                         uint64_t n, void* ws, size_t ws_bytes, cudaStream_t stream) {
  return launch_pair_pass<2>(k_cfgzero_final, "cfg-zero* scale", s_out, ec, eu, model_dtype, per_sample, n, ws,
                             ws_bytes, stream);
}

int launch_tcfg_words(float* w_out, const void* ec, const void* eu, int model_dtype, uint64_t per_sample, uint64_t n,
                      void* ws, size_t ws_bytes, cudaStream_t stream) {
  return launch_pair_pass<3>(k_tcfg_final, "tcfg words", w_out, ec, eu, model_dtype, per_sample, n, ws, ws_bytes,
                             stream);
}

// ---- Perp-Neg (dpm_perpneg_words; Armandpour, Sadeghian, Zheng, Sadeghian and Zhou, arXiv:2304.04968) -------------
// Over u = e_uncond and e_1..e_K, d_k = e_k - u in fp64 and the K fp64 sums N = ||d_1||^2, P_k = <d_k, d_1>
// (k = 2..K). k_perpneg_final then folds the sums with the host scales into one word per sample,
// w_1 = fl32(s_1 - s_2*c_2 - ... - s_K*c_K), c_k = P_k/N (0 when N == 0), which dpm_step_multi_masked reads as condition
// 1's period-1 weight map. Algorithmic bytes: (K+1)*s_model per element. The partials are K per chunk; the workspace
// is sized for kPNMax, whatever K is.
constexpr int kPNMax = 4;   // DPM_MAX_CONDITIONS

struct PNParams {
  WordsGeom g;           // partial: [n_samples * chunks][K]: N, P_2 .. P_K
  const void* eu;
  const void* ec[kPNMax];
  float* w_out;          // [n_samples]
  int32_t model_dtype;
  int32_t n_cond;
  float scales[kPNMax];  // fl32(s_1) .. fl32(s_K)
};

template <int K>
struct PerpNegPass {
  static_assert(K >= 2 && K <= kPNMax, "two to four conditions");
  using Params = PNParams;
  static constexpr int kSums = K, kWorkspaceSums = kPNMax;
  static constexpr bool kState = false;
  template <typename TE, typename TS, bool VEC>
  __device__ static void sums(const Params& p, const Chunk& c, double* warp_part, double (&s)[kSums]) {
    sums_over<TE, VEC>(p, c, warp_part, s, std::make_index_sequence<K>{});
  }
  template <typename TE, bool VEC, size_t... k>
  __device__ static void sums_over(const Params& p, const Chunk& c, double* warp_part, double (&s)[kSums],
                                   std::index_sequence<k...>) {
    double t[K];   // N, P_2 .. P_K
#pragma unroll
    for (int j = 0; j < K; ++j) t[j] = 0.0;
    visit<VEC>(c, nullptr, [&](int, int, const float (&v)[K + 1]) {
      const double d1 = (double)v[1] - (double)v[0];
      t[0] += d1 * d1;
#pragma unroll
      for (int j = 1; j < K; ++j) t[j] += ((double)v[j + 1] - (double)v[0]) * d1;
    }, In<TE>{p.eu, p.model_dtype}, In<TE>{p.ec[k], p.model_dtype}...);
#pragma unroll
    for (int j = 0; j < K; ++j) s[j] = cta_sum(t[j], warp_part);
  }
};

// The word of sample b from its merged sums, in fp64 left to right with each op rounded: t = s_1, then
// t = t - s_k*c_k for k = 2..K, rounded to fp32 once. A sum that is not finite gives k_tcfg_final's NaN.
__global__ void __launch_bounds__(kWThreads) k_perpneg_final(const __grid_constant__ PNParams p) {
  const uint64_t b = (uint64_t)blockIdx.x * kWThreads + threadIdx.x;
  if (b >= p.g.n_samples) return;
  const int K = p.n_cond;
  double s[kPNMax];
  merge_sums(p.g, b, K, s);
  bool finite = true;
#pragma unroll
  for (int k = 0; k < kPNMax; ++k)
    if (k < K) finite = finite && isfinite(s[k]);
  float w = __int_as_float(0x7fffffff);
  if (finite) {
    double t = (double)p.scales[0];
#pragma unroll
    for (int k = 1; k < kPNMax; ++k) {
      if (k < K) {
        const double ck = s[0] == 0.0 ? 0.0 : s[k] / s[0];
        t = t - (double)p.scales[k] * ck;
      }
    }
    w = (float)t;
  }
  p.w_out[b] = w;
}

int launch_perpneg_words(float* w_out, const void* eu, const void* const* ec, const float* scales, int n_cond,
                         int model_dtype, uint64_t per_sample, uint64_t n, void* ws, size_t ws_bytes,
                         cudaStream_t stream) {
  PNParams p;
  memset(&p, 0, sizeof(p));
  p.g.per_sample = per_sample; p.g.n_samples = n / per_sample;
  p.eu = eu; p.w_out = w_out; p.model_dtype = model_dtype; p.n_cond = n_cond;
  for (int k = 0; k < n_cond; ++k) { p.ec[k] = ec[k]; p.scales[k] = scales[k]; }
  const int md = model_dtype;
  const auto launch = n_cond == 2 ? launch_words<PerpNegPass<2>>
                      : n_cond == 3 ? launch_words<PerpNegPass<3>> : launch_words<PerpNegPass<4>>;
  return launch("perpneg words", p, k_perpneg_final, md, md,
                {{eu, md}, {p.ec[0], md}, {p.ec[1], md}, {p.ec[2], md}, {p.ec[3], md}}, ws, ws_bytes, stream);
}

}  // namespace dpm
