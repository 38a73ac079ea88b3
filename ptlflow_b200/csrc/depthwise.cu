// Depthwise k x k convolution fused with the residual and the GELU of SKFlow's PCBlock (skflow/update.py:32-33):
//   out[p, c] = gelu(x[p, c] + bias[c] + sum_{ky, kx} w[ky][kx][c] * x[p + (ky - k/2, kx - k/2), c])
// CUDA-core work (one multiply-add per tap and channel, nothing for the tensor cores to share).  A CTA owns an 8 x 16 pixel
// tile of CC channels: the tile plus its halo is staged once in shared memory as fp32 (zero outside the image, which is the
// "same" padding), next to the fp32 weights of those channels.  A thread owns a channel pair and a strip of R = 8 consecutive
// pixels of one row; per filter row it loads the R + k - 1 input pairs of that row once into registers and slides the k taps
// over them, so every staged value is read from shared memory k times fewer than a per-output loop would.  The epilogue is one of
// the kDw* modes: without the residual and the GELU (kDwBias) the same kernel is the first pass of pfb_depthwise_conv_layernorm
// below; kDwBiasGelu and kDwBiasAddend are the two depthwise convolutions of CCMR's LPI (pfb_depthwise_conv3x3_ex).
#include <atomic>

#include "common.cuh"

namespace pfb {

template <typename T> struct Pair;
template <> struct Pair<float> {
  using V = float2;
  static __device__ __forceinline__ float2 f2(V v) { return v; }
  static __device__ __forceinline__ V from(float a, float b) { return make_float2(a, b); }
};
template <> struct Pair<__half> {
  using V = __half2;
  static __device__ __forceinline__ float2 f2(V v) { return __half22float2(v); }
  static __device__ __forceinline__ V from(float a, float b) { return __floats2half2_rn(a, b); }
};
template <> struct Pair<__nv_bfloat16> {
  using V = __nv_bfloat162;
  static __device__ __forceinline__ float2 f2(V v) { return __bfloat1622float2(v); }
  static __device__ __forceinline__ V from(float a, float b) { return __floats2bfloat162_rn(a, b); }
};

constexpr int kDwTH = 8, kDwR = 8, kDwSX = 2, kDwTW = kDwR * kDwSX;  // output tile: 8 rows x 16 columns
// channels per CTA: 32 up to k = 15 (two CTAs of 110 KB per SM at k = 15); 8 above, where the halo tile grows quadratically
__host__ __device__ constexpr int dw_cc(int K) { return K <= 15 ? 32 : 8; }
__host__ __device__ constexpr int dw_threads(int K) { return dw_cc(K) / 2 * kDwSX * kDwTH; }
__host__ __device__ constexpr size_t dw_smem(int K) {
  return ((size_t)(kDwTH + K - 1) * (kDwTW + K - 1) + (size_t)K * K) * dw_cc(K) * sizeof(float);
}

// epilogues: y = dw(x) + bias, then  kDwBias: y;  kDwResidualGelu: gelu(x + y);  kDwBiasGelu: gelu(y);  kDwBiasAddend: y + addend
enum { kDwBias = 0, kDwResidualGelu = 1, kDwBiasGelu = 2, kDwBiasAddend = 3 };

template <typename T, int K, int kMode>
__global__ void __launch_bounds__(dw_threads(K)) depthwise_gelu_kernel(const T* __restrict__ x, int in_stride, T* __restrict__ out,
                                                                      int out_stride, const float* __restrict__ wgt,
                                                                      const float* __restrict__ bias, int H, int W, int C, int tiles_x,
                                                                      const T* __restrict__ addend, int addend_stride) {
  constexpr int CC = dw_cc(K), NP = CC / 2, THR = dw_threads(K);
  constexpr int PH = kDwTH + K - 1, PW = kDwTW + K - 1;
  using V = typename Pair<T>::V;
  extern __shared__ __align__(16) float dw_sm[];
  float* s_in = dw_sm;                 // [PH][PW][CC]
  float* s_w = dw_sm + PH * PW * CC;   // [K*K][CC]
  const int tile = blockIdx.x, c0 = blockIdx.y * CC, b = blockIdx.z;
  const int y0 = (tile / tiles_x) * kDwTH, x0 = (tile % tiles_x) * kDwTW;
  const int tid = threadIdx.x;

  for (int i = tid; i < K * K * NP; i += THR) {
    const int tap = i / NP, cp = i - tap * NP, c = c0 + 2 * cp;
    float2 w = make_float2(0.f, 0.f);
    if (c < C) w = make_float2(wgt[(size_t)tap * C + c], wgt[(size_t)tap * C + c + 1]);
    reinterpret_cast<float2*>(s_w)[i] = w;
  }
  const size_t img = (size_t)b * H * W;
  for (int i = tid; i < PH * PW * NP; i += THR) {
    const int cp = i % NP, pix = i / NP;
    const int iy = y0 - K / 2 + pix / PW, ix = x0 - K / 2 + pix % PW, c = c0 + 2 * cp;
    float2 v = make_float2(0.f, 0.f);
    if (iy >= 0 && iy < H && ix >= 0 && ix < W && c < C)
      v = Pair<T>::f2(*reinterpret_cast<const V*>(x + (img + (size_t)iy * W + ix) * in_stride + c));
    reinterpret_cast<float2*>(s_in)[i] = v;
  }
  __syncthreads();

  const int cp = tid % NP, sx = (tid / NP) % kDwSX, ty = tid / (NP * kDwSX);
  float2 acc[kDwR];
#pragma unroll
  for (int r = 0; r < kDwR; ++r) acc[r] = make_float2(0.f, 0.f);
  const float2* in2 = reinterpret_cast<const float2*>(s_in);
  const float2* w2 = reinterpret_cast<const float2*>(s_w);
#pragma unroll 1
  for (int ky = 0; ky < K; ++ky) {
    const float2* row = in2 + ((ty + ky) * PW + sx * kDwR) * NP + cp;
    float2 win[kDwR + K - 1];
#pragma unroll
    for (int j = 0; j < kDwR + K - 1; ++j) win[j] = row[j * NP];
#pragma unroll
    for (int kx = 0; kx < K; ++kx) {
      const float2 w = w2[(ky * K + kx) * NP + cp];
#pragma unroll
      for (int r = 0; r < kDwR; ++r) {
        acc[r].x = fmaf(win[r + kx].x, w.x, acc[r].x);
        acc[r].y = fmaf(win[r + kx].y, w.y, acc[r].y);
      }
    }
  }
  const int c = c0 + 2 * cp, oy = y0 + ty;
  if (c >= C || oy >= H) return;
  const float b0 = bias[c], b1 = bias[c + 1];
#pragma unroll
  for (int r = 0; r < kDwR; ++r) {
    const int ox = x0 + sx * kDwR + r;
    if (ox < W) {
      V* o = reinterpret_cast<V*>(out + (img + (size_t)oy * W + ox) * out_stride + c);
      if (kMode == kDwResidualGelu) {
        const float2 xc = in2[((ty + K / 2) * PW + sx * kDwR + r + K / 2) * NP + cp];  // the residual: the centre tap's input
        *o = Pair<T>::from(gelu_f32(xc.x + (acc[r].x + b0)), gelu_f32(xc.y + (acc[r].y + b1)));
      } else if (kMode == kDwBiasGelu) {
        *o = Pair<T>::from(gelu_f32(acc[r].x + b0), gelu_f32(acc[r].y + b1));
      } else if (kMode == kDwBiasAddend) {
        const float2 a = Pair<T>::f2(*reinterpret_cast<const V*>(addend + (img + (size_t)oy * W + ox) * addend_stride + c));
        *o = Pair<T>::from((acc[r].x + b0) + a.x, (acc[r].y + b1) + a.y);
      } else {
        *o = Pair<T>::from(acc[r].x + b0, acc[r].y + b1);
      }
    }
  }
}

template <typename T, int K, int kMode = kDwResidualGelu>
static int launch_dw(const T* x, int in_stride, T* out, int out_stride, const float* w, const float* bias, int B, int H, int W, int C,
                     cudaStream_t s, const T* addend = nullptr, int addend_stride = 0) {
  static std::atomic<unsigned long long> attr_done{0};
  const size_t smem = dw_smem(K);
  int dev = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  if (smem > 48 * 1024 && !(attr_done.load(std::memory_order_acquire) & (1ull << (dev & 63)))) {
    PFB_CUDA(cudaFuncSetAttribute(depthwise_gelu_kernel<T, K, kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
  }
  const int tiles_x = ceil_div(W, kDwTW), tiles_y = ceil_div(H, kDwTH);
  dim3 grid(tiles_x * tiles_y, ceil_div(C, dw_cc(K)), B);
  ProfScope prof(kMode == kDwBias ? KC_DW_LAYERNORM : KC_DEPTHWISE, s);
  depthwise_gelu_kernel<T, K, kMode><<<grid, dw_threads(K), smem, s>>>(x, in_stride, out, out_stride, w, bias, H, W, C, tiles_x, addend,
                                                                       addend_stride);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

template <typename T>
static int dispatch_dw(const T* x, int in_stride, T* out, int out_stride, const float* w, const float* bias, int B, int H, int W, int C,
                       int k, cudaStream_t s) {
  switch (k) {
#define PFB_DW_CASE(K) \
  case K: return launch_dw<T, K>(x, in_stride, out, out_stride, w, bias, B, H, W, C, s);
    PFB_DW_CASE(1) PFB_DW_CASE(3) PFB_DW_CASE(5) PFB_DW_CASE(7) PFB_DW_CASE(9) PFB_DW_CASE(11) PFB_DW_CASE(13) PFB_DW_CASE(15)
    PFB_DW_CASE(17) PFB_DW_CASE(19) PFB_DW_CASE(21) PFB_DW_CASE(23) PFB_DW_CASE(25) PFB_DW_CASE(27) PFB_DW_CASE(29) PFB_DW_CASE(31)
#undef PFB_DW_CASE
    default: break;
  }
  set_error("depthwise_conv_gelu: kernel size %d (odd, 1..31)", k);
  return PFB_ERR_ARG;
}

// ------------------------------------------------------------------------------------------------
// Depthwise k x k convolution + LayerNorm over the channels (SEA-RAFT's ConvNextBlock, sea_raft/layer.py:71-75) as two passes:
// the halo-tiled depthwise kernel above without its residual and GELU, y = dw_k(x) + bias, stored in the storage type, then a row
// LayerNorm over each pixel's C channels, in place.  Measured against a fused kernel that kept all channels of an 8-pixel strip in
// registers and read its window straight from global memory (DESIGN.md section 5): the fused kernel saved the round trip of y
// but took 1.4-1.5x as long at the config-3 grid, because it staged nothing in shared memory.
constexpr int kLnMaxC = 512;

// Row LayerNorm, in place allowed: one warp per pixel, lane l holds the channel pairs 2l + 64j in registers, mean then the variance
// about it by warp shuffles; the affine gamma / beta (fp32 [C]) when gamma is not NULL.
template <typename T>
__global__ void __launch_bounds__(256) layernorm_rows_kernel(const T* y, int in_stride, T* out, int out_stride, size_t P, int C, float eps,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta) {
  using V = typename Pair<T>::V;
  constexpr int NJ = kLnMaxC / 64;
  const size_t p = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= P) return;
  float2 v[NJ];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = 2 * lane + 64 * j;
    v[j] = c < C ? Pair<T>::f2(*reinterpret_cast<const V*>(y + p * in_stride + c)) : make_float2(0.f, 0.f);
    s += v[j].x + v[j].y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mu = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j)
    if (2 * lane + 64 * j < C) q += (v[j].x - mu) * (v[j].x - mu) + (v[j].y - mu) * (v[j].y - mu);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rs = rsqrtf(q / (float)C + eps);
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = 2 * lane + 64 * j;
    if (c >= C) continue;
    float2 n = make_float2((v[j].x - mu) * rs, (v[j].y - mu) * rs);
    if (gamma) n = make_float2(fmaf(n.x, gamma[c], beta[c]), fmaf(n.y, gamma[c + 1], beta[c + 1]));
    *reinterpret_cast<V*>(out + p * out_stride + c) = Pair<T>::from(n.x, n.y);
  }
}

template <typename T>
static int launch_dwln(const T* x, int in_stride, T* out, int out_stride, const float* w, const float* bias, int B, int H, int W, int C,
                       int k, float eps, cudaStream_t s) {
  int rc = PFB_ERR_ARG;
  switch (k) {
#define PFB_DWS_CASE(K) \
  case K: rc = launch_dw<T, K, kDwBias>(x, in_stride, out, out_stride, w, bias, B, H, W, C, s); break;
    PFB_DWS_CASE(1) PFB_DWS_CASE(3) PFB_DWS_CASE(5) PFB_DWS_CASE(7) PFB_DWS_CASE(9) PFB_DWS_CASE(11) PFB_DWS_CASE(13)
    PFB_DWS_CASE(15) PFB_DWS_CASE(17) PFB_DWS_CASE(19) PFB_DWS_CASE(21) PFB_DWS_CASE(23) PFB_DWS_CASE(25) PFB_DWS_CASE(27)
    PFB_DWS_CASE(29) PFB_DWS_CASE(31)
#undef PFB_DWS_CASE
    default: set_error("depthwise_conv_layernorm: kernel size %d (odd, 1..31)", k); break;
  }
  if (rc != PFB_OK) return rc;
  const size_t P = (size_t)B * H * W;
  ProfScope prof(KC_DW_LAYERNORM, s);
  layernorm_rows_kernel<T><<<(unsigned)ceil_div_sz(P, 8), 256, 0, s>>>(out, out_stride, out, out_stride, P, C, eps, nullptr, nullptr);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_depthwise_conv_layernorm(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset,
                                                    const float* weight, const float* bias, int B, int H, int W, int C, int k, float eps,
                                                    pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && out && weight && bias, "depthwise_conv_layernorm: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "depthwise_conv_layernorm: bad dtype");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 2 == 0 && C <= kLnMaxC,
                "depthwise_conv_layernorm: bad shape %dx%dx%dx%d (C even, <= %d)", B, H, W, C, kLnMaxC);
  PFB_CHECK_ARG(B <= 65535, "depthwise_conv_layernorm: batch %d too large", B);
  PFB_CHECK_ARG((k & 1) && k >= 1 && k <= 31, "depthwise_conv_layernorm: kernel size %d (odd, 1..31)", k);
  PFB_CHECK_ARG(eps > 0.f, "depthwise_conv_layernorm: eps must be positive");
  PFB_CHECK_ARG(in_offset >= 0 && out_offset >= 0 && in_stride >= in_offset + C && out_stride >= out_offset + C &&
                    in_offset % 2 == 0 && out_offset % 2 == 0 && in_stride % 2 == 0 && out_stride % 2 == 0,
                "depthwise_conv_layernorm: strides / offsets must be even and hold C channels");
  const size_t es = dtype_size(dtype);
  const char* xb = reinterpret_cast<const char*>(x) + (size_t)in_offset * es;
  char* ob = reinterpret_cast<char*>(out) + (size_t)out_offset * es;
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(xb) % (2 * es)) == 0 && (reinterpret_cast<uintptr_t>(ob) % (2 * es)) == 0,
                "depthwise_conv_layernorm: misaligned channel pairs");
  cudaStream_t s = as_stream(stream);
  PFB_DISPATCH_DTYPE(dtype, T, {
    return launch_dwln<T>(reinterpret_cast<const T*>(xb), in_stride, reinterpret_cast<T*>(ob), out_stride, weight, bias, B, H, W, C, k,
                          eps, s);
  });
  return PFB_ERR_ARG;
}

extern "C" PFB_API int pfb_depthwise_conv_gelu(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset,
                                               const float* weight, const float* bias, int B, int H, int W, int C, int k, pfb_dtype dtype,
                                               pfb_stream stream) {
  PFB_CHECK_ARG(x && out && weight && bias, "depthwise_conv_gelu: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "depthwise_conv_gelu: bad dtype");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 2 == 0, "depthwise_conv_gelu: bad shape %dx%dx%dx%d (C must be even)", B, H, W, C);
  PFB_CHECK_ARG((k & 1) && k >= 1 && k <= 31, "depthwise_conv_gelu: kernel size %d (odd, 1..31)", k);
  PFB_CHECK_ARG(in_offset >= 0 && out_offset >= 0 && in_stride >= in_offset + C && out_stride >= out_offset + C &&
                    in_offset % 2 == 0 && out_offset % 2 == 0 && in_stride % 2 == 0 && out_stride % 2 == 0,
                "depthwise_conv_gelu: strides / offsets must be even and hold C channels");
  const size_t es = dtype_size(dtype);
  const char* xb = reinterpret_cast<const char*>(x) + (size_t)in_offset * es;
  char* ob = reinterpret_cast<char*>(out) + (size_t)out_offset * es;
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(xb) % (2 * es)) == 0 && (reinterpret_cast<uintptr_t>(ob) % (2 * es)) == 0,
                "depthwise_conv_gelu: misaligned channel pairs");
  cudaStream_t s = as_stream(stream);
  PFB_DISPATCH_DTYPE(dtype, T, {
    return dispatch_dw<T>(reinterpret_cast<const T*>(xb), in_stride, reinterpret_cast<T*>(ob), out_stride, weight, bias, B, H, W, C, k, s);
  });
  return PFB_ERR_ARG;
}

// ---- a18: CCMR's XCiT block (ccmr/xcit.py:98-139, 242-300) ----
extern "C" PFB_API int pfb_layernorm(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset, const float* gamma,
                                     const float* beta, size_t P, int C, float eps, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && out, "layernorm: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "layernorm: bad dtype");
  PFB_CHECK_ARG(P > 0 && C > 0 && C % 2 == 0 && C <= kLnMaxC, "layernorm: bad shape P=%zu C=%d (C even, <= %d)", P, C, kLnMaxC);
  PFB_CHECK_ARG((gamma == nullptr) == (beta == nullptr), "layernorm: gamma and beta must both be set or both be NULL");
  PFB_CHECK_ARG(eps > 0.f, "layernorm: eps must be positive");
  PFB_CHECK_ARG(in_offset >= 0 && out_offset >= 0 && in_stride >= in_offset + C && out_stride >= out_offset + C && in_offset % 2 == 0 &&
                    out_offset % 2 == 0 && in_stride % 2 == 0 && out_stride % 2 == 0,
                "layernorm: strides / offsets must be even and hold C channels");
  const size_t es = dtype_size(dtype);
  const char* xb = reinterpret_cast<const char*>(x) + (size_t)in_offset * es;
  char* ob = reinterpret_cast<char*>(out) + (size_t)out_offset * es;
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(xb) % (2 * es)) == 0 && (reinterpret_cast<uintptr_t>(ob) % (2 * es)) == 0,
                "layernorm: misaligned channel pairs");
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_DW_LAYERNORM, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    layernorm_rows_kernel<T><<<(unsigned)ceil_div_sz(P, 8), 256, 0, s>>>(reinterpret_cast<const T*>(xb), in_stride, reinterpret_cast<T*>(ob),
                                                                        out_stride, P, C, eps, gamma, beta);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_depthwise_conv3x3_ex(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset,
                                                const float* weight, const float* bias, const void* addend, int addend_stride,
                                                int addend_offset, int B, int H, int W, int C, int mode, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && out && weight && bias, "depthwise_conv3x3_ex: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && (mode == 0 || mode == 1), "depthwise_conv3x3_ex: bad dtype or mode %d", mode);
  PFB_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && W > 0 && C > 0 && C % 2 == 0, "depthwise_conv3x3_ex: bad shape %dx%dx%dx%d (C even)", B, H,
                W, C);
  PFB_CHECK_ARG(in_offset >= 0 && out_offset >= 0 && in_stride >= in_offset + C && out_stride >= out_offset + C && in_offset % 2 == 0 &&
                    out_offset % 2 == 0 && in_stride % 2 == 0 && out_stride % 2 == 0,
                "depthwise_conv3x3_ex: strides / offsets must be even and hold C channels");
  if (mode == 1)
    PFB_CHECK_ARG(addend && addend_offset >= 0 && addend_offset % 2 == 0 && addend_stride % 2 == 0 && addend_stride >= addend_offset + C,
                  "depthwise_conv3x3_ex: mode 1 needs an addend with an even stride / offset holding C channels");
  const size_t es = dtype_size(dtype);
  const char* xb = reinterpret_cast<const char*>(x) + (size_t)in_offset * es;
  char* ob = reinterpret_cast<char*>(out) + (size_t)out_offset * es;
  const char* ab = mode == 1 ? reinterpret_cast<const char*>(addend) + (size_t)addend_offset * es : nullptr;
  PFB_CHECK_ARG(((reinterpret_cast<uintptr_t>(xb) | reinterpret_cast<uintptr_t>(ob) | reinterpret_cast<uintptr_t>(ab)) % (2 * es)) == 0,
                "depthwise_conv3x3_ex: misaligned channel pairs");
  cudaStream_t s = as_stream(stream);
  PFB_DISPATCH_DTYPE(dtype, T, {
    const T* xt = reinterpret_cast<const T*>(xb);
    T* ot = reinterpret_cast<T*>(ob);
    if (mode == 0) return launch_dw<T, 3, kDwBiasGelu>(xt, in_stride, ot, out_stride, weight, bias, B, H, W, C, s);
    return launch_dw<T, 3, kDwBiasAddend>(xt, in_stride, ot, out_stride, weight, bias, B, H, W, C, s, reinterpret_cast<const T*>(ab),
                                          addend_stride);
  });
  return PFB_ERR_ARG;
}
