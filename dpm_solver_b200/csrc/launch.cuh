// launch.cuh -- host-side helpers shared by the translation units of libdpmsolver_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"

namespace dpm {

struct Tuning {
  int variant;      // 0 direct, 1 TMA ring
  int threads;      // threads per CTA (0 = default)
  int ctas_per_sm;  // persistent-grid CTAs per SM (0 = default)
};

int sm_count();                     // SMs of the current device (cached per device)
int max_smem_optin();               // max opt-in dynamic shared memory per CTA
void count_launch();                // bump the library launch counter
// opt the kernel into the device's maximum dynamic shared memory (and, optionally, non-portable
// cluster sizes) the first time it is used on the current device; later calls are a hash lookup
int ensure_max_smem(const void* kernel, bool nonportable_cluster = false);
void set_error(const char* fmt, ...);
int launch_error(const char* what, cudaError_t e);   // records "what: <CUDA error>", clears it, returns its code

// ---- runtime -> compile-time dispatch of the kernel pickers ----------------------------------------
template <typename TE_, typename TS_> struct PacketPair {
  using TE = TE_;   // network output
  using TS = TS_;   // state and buffers
};
// Calls f(PacketPair<TE, TS>{}) for a runtime (model dtype, state dtype) that is one of the five pairs the packet
// kernels are built for: f32/f32, bf16/bf16, f16/f16, bf16->f32, f16->f32. Other pairs give a value-initialised result.
template <typename F>
static inline auto with_packet_pair(int md, int sd, F&& f) -> decltype(f(PacketPair<float, float>{})) {
  if (md == DPM_F32 && sd == DPM_F32) return f(PacketPair<float, float>{});
  if (md == DPM_BF16 && sd == DPM_BF16) return f(PacketPair<__nv_bfloat16, __nv_bfloat16>{});
  if (md == DPM_F16 && sd == DPM_F16) return f(PacketPair<__half, __half>{});
  if (md == DPM_BF16 && sd == DPM_F32) return f(PacketPair<__nv_bfloat16, float>{});
  if (md == DPM_F16 && sd == DPM_F32) return f(PacketPair<__half, float>{});
  return {};
}
// Calls f(std::integral_constant<int, FORM>{}) for a runtime dpm_form. Other values give a value-initialised result.
template <typename F>
static inline auto with_form(int form, F&& f) -> decltype(f(std::integral_constant<int, DPM_FORM_NONE>{})) {
  switch (form) {
    case DPM_FORM_NONE: return f(std::integral_constant<int, DPM_FORM_NONE>{});
    case DPM_FORM_LIN1: return f(std::integral_constant<int, DPM_FORM_LIN1>{});
    case DPM_FORM_LIN2: return f(std::integral_constant<int, DPM_FORM_LIN2>{});
    case DPM_FORM_LIN3: return f(std::integral_constant<int, DPM_FORM_LIN3>{});
    case DPM_FORM_DIFF2: return f(std::integral_constant<int, DPM_FORM_DIFF2>{});
    case DPM_FORM_MS3: return f(std::integral_constant<int, DPM_FORM_MS3>{});
    case DPM_FORM_SS3T: return f(std::integral_constant<int, DPM_FORM_SS3T>{});
  }
  return {};
}
// The step kernel pick(PacketPair<TE, TS>{}, NE, FORM) names for a launch (NE and FORM as std::integral_constant).
// A launch without network outputs (NE == 0) reads state-typed streams only: it is served by the same-type pairs
// (TE = TS, picked by the state dtype), and not for FORM_NONE, which would compute nothing.
template <typename R, typename Pick>
static inline R pick_step(const KParams& p, Pick&& pick) {
  const int md = p.n_model == 0 ? p.state_dtype : p.model_dtype;
  return with_packet_pair(md, p.state_dtype, [&](auto pair) -> R {
    return with_form(p.form, [&](auto form) -> R {
      using Pair = decltype(pair);
      switch (p.n_model) {
        case 0:
          if constexpr (decltype(form)::value != DPM_FORM_NONE && std::is_same_v<typename Pair::TE, typename Pair::TS>)
            return pick(pair, std::integral_constant<int, 0>{}, form);
          return R{};
        case 1: return pick(pair, std::integral_constant<int, 1>{}, form);
        case 2: return pick(pair, std::integral_constant<int, 2>{}, form);
      }
      return R{};
    });
  });
}

// Programmatic dependent launch (PDL): the step kernels call pdl_wait() after their prologue (barrier init, index
// setup) and before touching global memory, and pdl_trigger() at entry; launched with the programmatic-stream-
// serialization attribute, the CTAs of step i+1 become resident while step i drains and only their first global
// access waits for its completion (and visibility). Without the attribute both are no-ops. The dependent grid starts
// only once every CTA of the primary has run pdl_trigger(), i.e. once the primary's last wave is resident, so an
// early dependent can never starve its primary, whatever the number of waves.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
bool pdl_enabled();   // DPM_PDL=0 turns the launch attribute off (A/B measurements)

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), unsigned grid, unsigned block, size_t smem, cudaStream_t stream,
                                     Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid, 1, 1);
  cfg.blockDim = dim3(block, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// each returns 0 on launch, 1 if this variant does not serve the request, <0 / cudaError on error
int launch_step_direct(const KParams& p, const Tuning& t, cudaStream_t stream);
int launch_step_scalar(const KParams& p, cudaStream_t stream);
int launch_step_tma(const KParams& p, const Tuning& t, cudaStream_t stream);
void philox_policy(uint64_t numel, uint32_t* grid, uint64_t* counter_offset);
int launch_noise_philox(void* out, const void* x, const void* xt, const float* mask, uint64_t mask_n, uint64_t n,
                        int t_count, const float* alpha, const float* sigma, uint64_t seed, uint64_t offset,
                        int x_dtype, int out_dtype, cudaStream_t stream);
int launch_adaptive_init(const dpm_adaptive_ctl* a, float t_T, float h_init, cudaStream_t stream);
int launch_adaptive_plan(const dpm_adaptive_ctl* a, cudaStream_t stream);
int launch_adaptive_decide(const dpm_adaptive_ctl* a, cudaStream_t stream);
int launch_select_copy(void* dst, const void* src, const float* state, uint64_t bytes, cudaStream_t stream);
int launch_duplicate(void* dst, const void* src, uint64_t bytes, cudaStream_t stream);
int launch_step_multi(const MultiParams& mp, const Tuning& t, cudaStream_t stream);
int launch_step_multi_scalar(const MultiParams& mp, cudaStream_t stream);
int launch_step_multi_masked(const MaskedParams& q, const Tuning& t, cudaStream_t stream);
int launch_step_multi_masked_scalar(const MaskedParams& q, cudaStream_t stream);
int launch_step_unipc(const UniParams& up, const Tuning& t, cudaStream_t stream);
int launch_step_unipc_scalar(const UniParams& up, cudaStream_t stream);
int launch_step_cfgpp(const CfgppParams& q, const Tuning& t, cudaStream_t stream);
int launch_step_cfgpp_scalar(const CfgppParams& q, cudaStream_t stream);
// one SDE-DPM-Solver++ update (step_sde.cu): p as dpm_step builds it plus the per-sample words; z NULL = drawn in-kernel
int launch_step_sde(const KParams& p, const float* z, float cz, uint64_t seed, uint64_t offset, bool aligned_all,
                    cudaStream_t stream);
int launch_replicate(void* dst, const void* src, uint64_t bytes, int copies, cudaStream_t stream);
int launch_quantile(float* s_out, const KParams& p, uint64_t n_samples, float q, float max_val,
                    void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t quantile_workspace_bytes(uint64_t n_samples, uint64_t per_sample);
size_t adaptive_workspace_bytes(uint64_t n, uint64_t per_sample);
int launch_adaptive_error(float* out, const void* xh, const void* xl, const void* xp, float atol, float rtol,
                          uint64_t per_sample, uint64_t n, int dtype, void* ws, size_t ws_bytes, cudaStream_t stream);
// the per-sample guidance words passes (words.cu): the workspace of `sums` fp64 partials per chunk of a sample
size_t words_workspace_bytes(uint64_t n_samples, uint64_t per_sample, int sums);
int launch_cfg_rescale_ratio(float* ratio, const void* ec, const void* eu, float guidance, uint64_t per_sample,
                             uint64_t n, int dtype, void* ws, size_t ws_bytes, cudaStream_t stream,
                             const float* gscale = nullptr);
int launch_apg_words(float* words, const KParams& kp, const float* gscale, float eta, float norm_threshold,
                     float momentum, const float* r_prev, float* r_out, void* ws, size_t ws_bytes, cudaStream_t stream);
int launch_cfgzero_scale(float* s_out, const void* ec, const void* eu, int model_dtype, uint64_t per_sample,
                         uint64_t n, void* ws, size_t ws_bytes, cudaStream_t stream);
int launch_tcfg_words(float* w_out, const void* ec, const void* eu, int model_dtype, uint64_t per_sample, uint64_t n,
                      void* ws, size_t ws_bytes, cudaStream_t stream);
int launch_perpneg_words(float* w_out, const void* eu, const void* const* ec, const float* scales, int n_cond,
                         int model_dtype, uint64_t per_sample, uint64_t n, void* ws, size_t ws_bytes,
                         cudaStream_t stream);
int fdg_supported(uint64_t H, uint64_t W, int levels, int model_dtype);
int launch_fdg_guided(void* g, const void* ec, const void* eu, int model_dtype, uint64_t planes, uint64_t H, uint64_t W,
                      int64_t sample_stride, int64_t plane_stride, int64_t h_stride, int64_t w_stride, int levels,
                      const float* scales, uint64_t scale_stride, uint64_t planes_per_sample, cudaStream_t stream);

}  // namespace dpm
