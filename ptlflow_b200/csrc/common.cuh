// Shared helpers for the ptlflow_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ptlflow_b200.h"

namespace pfb {

void set_error(const char* fmt, ...);

#define PFB_CHECK_ARG(cond, ...)           \
  do {                                     \
    if (!(cond)) {                         \
      ::pfb::set_error(__VA_ARGS__);       \
      return PFB_ERR_ARG;                  \
    }                                      \
  } while (0)

#define PFB_CUDA(call)                                                                        \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess) {                                                                 \
      ::pfb::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return PFB_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

#define PFB_LAUNCH_CHECK() PFB_CUDA(cudaPeekAtLastError())

inline size_t dtype_size(pfb_dtype dt) { return dt == PFB_F32 ? 4 : 2; }
inline bool dtype_ok(int dt) { return dt == PFB_F32 || dt == PFB_F16 || dt == PFB_BF16; }
inline cudaStream_t as_stream(pfb_stream s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- scalar conversions -----------------------------------------------------------
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// load element i of a buffer whose dtype is only known at run time (slow path helpers)
__device__ __forceinline__ float load_as_f32(const void* p, size_t i, int dt) {
  if (dt == PFB_F32) return reinterpret_cast<const float*>(p)[i];
  if (dt == PFB_F16) return __half2float(reinterpret_cast<const __half*>(p)[i]);
  return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}
__device__ __forceinline__ void store_from_f32(void* p, size_t i, int dt, float v) {
  if (dt == PFB_F32) reinterpret_cast<float*>(p)[i] = v;
  else if (dt == PFB_F16) reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
  else reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
}

__device__ __forceinline__ float sigmoid_f32(float x) { return 1.0f / (1.0f + expf(-x)); }
// exact (erf) GELU, the default of F.gelu / nn.GELU
__device__ __forceinline__ float gelu_f32(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// Dispatch a templated launcher on the storage dtype.
#define PFB_DISPATCH_DTYPE(dt, T, ...)                        \
  do {                                                        \
    if ((dt) == PFB_F32) { using T = float; __VA_ARGS__; }    \
    else if ((dt) == PFB_F16) { using T = __half; __VA_ARGS__; } \
    else { using T = __nv_bfloat16; __VA_ARGS__; }            \
  } while (0)

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline size_t ceil_div_sz(size_t a, size_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t a, size_t b) { return (a + b - 1) / b * b; }

// number of SMs of the current device (cached)
int sm_count();

// kernel classes for launch accounting / live per-class timing (prof.cu)
// ---- programmatic dependent launch (PDL) ------------------------------------------------------------------
// The refinement loop is ~25 short dependent launches per iteration; the kernel-to-kernel hand-over (grid drain,
// launch latency, prologue of the next kernel) is ~2 us each.  Kernels on that path are launched with
// programmaticStreamSerialization: they may be scheduled while the previous grid drains, do their data-independent
// prologue, and block in pdl_wait() until the previous grid has completed and flushed.  pdl_trigger() lets the
// NEXT kernel in the stream do the same relative to this one.  PFB_PDL=0 turns the attribute off.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
int pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

enum KernelClass { KC_VOLUME = 0, KC_POOL, KC_LOOKUP, KC_ONTHEFLY, KC_CONV, KC_UPSAMPLE, KC_MISC,
                   KC_ENC_AFFINE, KC_ENC_STATS, KC_ENC_CONV1, KC_FLOWCONV, KC_GATHER, KC_DEPTHWISE, KC_DW_LAYERNORM, KC_COUNT };
class ProfScope {
 public:
  ProfScope(int kc, cudaStream_t s);
  ~ProfScope();
 private:
  int kc_;
  cudaStream_t s_;
  void* a_;
};

// ---- kernel families implemented in the other translation units ---------------------
// conv_simt.cu
int conv2d_simt(const pfb_conv_params* p, cudaStream_t s);
// conv_umma.cu (wgmma); returns PFB_ERR_UNSUPPORTED when the shape does not fit
int conv2d_umma(const pfb_conv_params* p, cudaStream_t s);
bool conv2d_umma_supported(const pfb_conv_params* p);
// conv_special.cu
bool conv_cout2_supported(const pfb_conv_params* p);
int conv_cout2_flow(const pfb_conv_params* p, cudaStream_t s);
bool conv_flow7x7_supported(const pfb_conv_params* p);
int conv_flow7x7(const pfb_conv_params* p, cudaStream_t s);
// corr_umma.cu
int corr_volume_umma(const void* f1, const void* f2, void* const* pyr, int B, int N1, int H, int W, int C, int L, float scale,
                     pfb_dtype dt, cudaStream_t s);
bool corr_volume_umma_supported(int B, int H, int W, int C, int L, pfb_dtype dt);
// corr_onthefly_umma.cu
bool corr_onthefly_umma_supported(int B, int H, int W, int C, int levels, int radius, pfb_dtype dt, int out_stride);
// corr_umma.cu, tiled pyramid (layout: corr_tiled.cu)
int corr_volume_tiled(const void* f1, const void* f2, void* const* pyr, int B, int N1, int H, int W, int C, int L, float scale,
                      pfb_dtype dt, cudaStream_t s);
bool corr_volume_tiled_supported(int B, int H, int W, int C, int L, pfb_dtype dt);

}  // namespace pfb
