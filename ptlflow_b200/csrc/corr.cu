// Correlation volume (SIMT reference-precision path), pooled pyramid, multi-scale lookup and
// the on-the-fly lookup.  Reference semantics: ptlflow/models/raft/corr.py:13-101 and
// ptlflow/utils/external/alt_cuda_corr/correlation_kernel.cu:18-119 (re-designed, not ported:
// the reference kernel does 100 __syncthreads rounds per 32-channel chunk with RMW `+=` on
// global memory; here a warp owns a query, keeps its window in shared memory and writes once).
#include "common.cuh"

namespace pfb {

// =====================================================================================
// a1 (SIMT): C[b][n1][n2] = scale * sum_c F1[b][n1][c] * F2[b][n2][c]
// 64x64 output tile, 16-wide K slices, 256 threads x (4x4) micro tiles, fp32 accumulate.
// =====================================================================================
template <typename T>
__global__ void __launch_bounds__(256) corr_volume_simt_kernel(const T* __restrict__ f1, const T* __restrict__ f2,
                                                               T* __restrict__ out, int N1, int N2, int C, float scale) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int b = blockIdx.z;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int lrow = tid >> 2, lk = (tid & 3) * 4;  // loader: row 0..63, 4 consecutive channels
  const T* a_base = f1 + (size_t)b * N1 * C;
  const T* b_base = f2 + (size_t)b * N2 * C;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < C; k0 += BK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int k = k0 + lk + j;
      int ra = m0 + lrow, rb = n0 + lrow;
      As[lk + j][lrow] = (ra < N1 && k < C) ? to_f32(a_base[(size_t)ra * C + k]) : 0.f;
      Bs[lk + j][lrow] = (rb < N2 && k < C) ? to_f32(b_base[(size_t)rb * C + k]) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bb[j] = Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }
  T* o = out + (size_t)b * N1 * N2;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= N1) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n < N2) o[(size_t)m * N2 + n] = from_f32<T>(acc[i][j] * scale);
    }
  }
}

// =====================================================================================
// a2: 2x2 mean over the last two spatial axes of [N, H, W, C] -> [N, H/2, W/2, C]
// (C = 1 for the volume pyramid; C = feature channels for the on-the-fly feature pyramid).
// =====================================================================================
template <typename T>
__global__ void avg_pool2x2_kernel(const T* __restrict__ in, T* __restrict__ out, size_t total, int H, int W,
                                   int C) {
  const int Ho = H / 2, Wo = W / 2;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    int c = (int)(idx % C);
    size_t t = idx / C;
    int x = (int)(t % Wo);
    t /= Wo;
    int y = (int)(t % Ho);
    size_t n = t / Ho;
    const T* p = in + ((n * H + 2 * y) * (size_t)W + 2 * x) * C + c;
    float s = to_f32(p[0]) + to_f32(p[C]) + to_f32(p[(size_t)W * C]) + to_f32(p[(size_t)W * C + C]);
    out[idx] = from_f32<T>(0.25f * s);
  }
}

// =====================================================================================
// a3: lookup.  One warp per query pixel.  Per level the warp stages the (2r+2)^2 integer-tap
// window in shared memory (rows read with consecutive lanes on consecutive x), then blends:
// all (2r+1)^2 samples share the same fractional part.
// =====================================================================================
struct LevelTable {
  const void* ptr[PFB_MAX_LEVELS];
  int h[PFB_MAX_LEVELS];
  int w[PFB_MAX_LEVELS];
};

template <typename TO>
__device__ __forceinline__ void store_lookup(TO* out, int nchw, size_t q, int hw, int planes, int out_stride,
                                             int ch, float v) {
  if (nchw) {
    size_t b = q / hw, pix = q % hw;
    out[(b * planes + ch) * (size_t)hw + pix] = from_f32<TO>(v);
  } else {
    out[q * (size_t)out_stride + ch] = from_f32<TO>(v);
  }
}

template <typename T, typename TO>
__global__ void __launch_bounds__(128) corr_lookup_kernel(LevelTable lv, const float* __restrict__ coords,
                                                          TO* __restrict__ out, int nq, int hw, int levels,
                                                          int r, int nchw, int out_stride) {
  extern __shared__ float smem[];
  const int D = 2 * r + 2, K = 2 * r + 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* win = smem + warp * D * D;
  const int q = blockIdx.x * (blockDim.x >> 5) + warp;
  if (q >= nq) return;
  const float cx = coords[2 * (size_t)q], cy = coords[2 * (size_t)q + 1];
  const int planes = levels * K * K;
  for (int l = 0; l < levels; ++l) {
    const float s = 1.0f / (float)(1 << l);
    const float x = cx * s, y = cy * s;
    const int Hl = lv.h[l], Wl = lv.w[l];
    const bool finite = (fabsf(x) < 1e7f) && (fabsf(y) < 1e7f);
    const float xf = finite ? floorf(x) : -1e6f, yf = finite ? floorf(y) : -1e6f;
    const float fx = finite ? x - xf : 0.f, fy = finite ? y - yf : 0.f;
    const int x0 = (int)xf - r, y0 = (int)yf - r;
    const T* base = reinterpret_cast<const T*>(lv.ptr[l]) + (size_t)q * Hl * Wl;
    for (int t = lane; t < D * D; t += 32) {
      int j = t / D, i = t - j * D;  // j: y index (rows), i: x index (contiguous in memory)
      int xi = x0 + i, yi = y0 + j;
      float v = 0.f;
      if (xi >= 0 && xi < Wl && yi >= 0 && yi < Hl) v = to_f32(base[(size_t)yi * Wl + xi]);
      win[i * D + j] = v;
    }
    __syncwarp();
    const float w00 = (1.f - fx) * (1.f - fy), w10 = fx * (1.f - fy), w01 = (1.f - fx) * fy, w11 = fx * fy;
    for (int o = lane; o < K * K; o += 32) {
      int i = o / K, j = o - i * K;  // channel = i*K + j, i <-> x offset (x-major, corr.py:43-47)
      float v = w00 * win[i * D + j] + w10 * win[(i + 1) * D + j] + w01 * win[i * D + j + 1] +
                w11 * win[(i + 1) * D + j + 1];
      store_lookup<TO>(out, nchw, (size_t)q, hw, planes, out_stride, l * K * K + o, v);
    }
    __syncwarp();
  }
  // pixel-major output wider than the lookup: zero the pad columns (they meet zero weight rows)
  if (!nchw)
    for (int c = planes + lane; c < out_stride; c += 32) out[(size_t)q * out_stride + c] = from_f32<TO>(0.f);
}

// Fast path (radius <= 4, levels <= 4, pixel-major output): every lane issues the gathers of ALL levels
// before any is consumed (16 independent loads in flight per lane instead of 4 dependent rounds), the four
// windows live side by side in shared memory, and the L*(2r+1)^2 outputs are written as one coalesced run.
template <typename T, typename TO, int R>
__global__ void __launch_bounds__(128) corr_lookup_r4_kernel(LevelTable lv, const float* __restrict__ coords,
                                                             TO* __restrict__ out, int nq, int levels, int out_stride) {
  pdl_wait();     // coords / volume come from the previous kernels in the stream
  pdl_trigger();  // the next kernel may be scheduled while this grid drains
  __shared__ float smem[4][4 * 100];
  __shared__ float wts[4][4][4];
  // compile-time radius: every index division below becomes a multiply-shift
  constexpr int r = R, D = 2 * R + 2, K = 2 * R + 1, DD = D * D, KK = K * K;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* win = smem[warp];
  const int q = blockIdx.x * 4 + warp;
  if (q >= nq) return;
  const float cx = coords[2 * (size_t)q], cy = coords[2 * (size_t)q + 1];
  float vals[4][4];
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    if (l < levels) {
      const float s = 1.0f / (float)(1 << l);
      const float x = cx * s, y = cy * s;
      const int Hl = lv.h[l], Wl = lv.w[l];
      const bool finite = (fabsf(x) < 1e7f) && (fabsf(y) < 1e7f);
      const float xf = finite ? floorf(x) : -1e6f, yf = finite ? floorf(y) : -1e6f;
      const float fx = finite ? x - xf : 0.f, fy = finite ? y - yf : 0.f;
      if (lane == 0) {
        wts[warp][l][0] = (1.f - fx) * (1.f - fy);
        wts[warp][l][1] = fx * (1.f - fy);
        wts[warp][l][2] = (1.f - fx) * fy;
        wts[warp][l][3] = fx * fy;
      }
      const int x0 = (int)xf - r, y0 = (int)yf - r;
      const T* base = reinterpret_cast<const T*>(lv.ptr[l]) + (size_t)q * Hl * Wl;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int t = lane + 32 * k;
        const int j = t / D, i = t - j * D;
        const int xi = x0 + i, yi = y0 + j;
        float v = 0.f;
        if (t < DD && xi >= 0 && xi < Wl && yi >= 0 && yi < Hl) v = to_f32(__ldg(base + (size_t)yi * Wl + xi));
        vals[l][k] = v;
      }
    }
  }
#pragma unroll
  for (int l = 0; l < 4; ++l) {
    if (l < levels) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int t = lane + 32 * k;
        const int j = t / D, i = t - j * D;
        if (t < DD) win[l * 100 + i * D + j] = vals[l][k];
      }
    }
  }
  __syncwarp();
  const int planes = levels * KK;
  TO* o = out + (size_t)q * out_stride;
  for (int c = lane; c < planes; c += 32) {
    const int l = c / KK, rem = c - l * KK;
    const int i = rem / K, j = rem - i * K;
    const float* w = win + l * 100;
    const float* ww = wts[warp][l];
    o[c] = from_f32<TO>(ww[0] * w[i * D + j] + ww[1] * w[(i + 1) * D + j] + ww[2] * w[i * D + j + 1] + ww[3] * w[(i + 1) * D + j + 1]);
  }
  for (int c = planes + lane; c < out_stride; c += 32) o[c] = from_f32<TO>(0.f);
}

// =====================================================================================
// a4: on-the-fly lookup.  One warp per query; the query's feature vector sits in shared memory
// as fp32; each lane owns integer taps of the window and runs the full C-long dot product with
// 128-bit loads of the target pixel's channel vector.
// =====================================================================================
template <typename T>
__device__ __forceinline__ float dot_row(const T* __restrict__ g, const float* __restrict__ s, int C);

template <>
__device__ __forceinline__ float dot_row<float>(const float* __restrict__ g, const float* __restrict__ s, int C) {
  float acc = 0.f;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int c = 0; c < C / 4; ++c) {
    float4 v = __ldg(g4 + c);
    acc = fmaf(v.x, s[4 * c], acc);
    acc = fmaf(v.y, s[4 * c + 1], acc);
    acc = fmaf(v.z, s[4 * c + 2], acc);
    acc = fmaf(v.w, s[4 * c + 3], acc);
  }
  return acc;
}
template <>
__device__ __forceinline__ float dot_row<__half>(const __half* __restrict__ g, const float* __restrict__ s, int C) {
  float acc = 0.f;
  const uint4* g4 = reinterpret_cast<const uint4*>(g);
  for (int c = 0; c < C / 8; ++c) {
    uint4 v = __ldg(g4 + c);
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 f = __half22float2(h[k]);
      acc = fmaf(f.x, s[8 * c + 2 * k], acc);
      acc = fmaf(f.y, s[8 * c + 2 * k + 1], acc);
    }
  }
  return acc;
}
template <>
__device__ __forceinline__ float dot_row<__nv_bfloat16>(const __nv_bfloat16* __restrict__ g,
                                                        const float* __restrict__ s, int C) {
  float acc = 0.f;
  const uint4* g4 = reinterpret_cast<const uint4*>(g);
  for (int c = 0; c < C / 8; ++c) {
    uint4 v = __ldg(g4 + c);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 f = __bfloat1622float2(h[k]);
      acc = fmaf(f.x, s[8 * c + 2 * k], acc);
      acc = fmaf(f.y, s[8 * c + 2 * k + 1], acc);
    }
  }
  return acc;
}

template <typename T, typename TO>
__global__ void __launch_bounds__(128) corr_onthefly_kernel(const T* __restrict__ fmap1, LevelTable lv,
                                                            const float* __restrict__ coords,
                                                            TO* __restrict__ out, int nq, int hw, int C,
                                                            int levels, int r, float scale, int nchw,
                                                            int out_stride, const unsigned char* __restrict__ flags) {
  extern __shared__ float smem[];
  const int D = 2 * r + 2, K = 2 * r + 1;
  const int warps = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* qv = smem + warp * C;                      // query feature vector, fp32
  float* win = smem + warps * C + warp * D * D;     // window of raw dot products
  const int q = blockIdx.x * warps + warp;
  if (q >= nq) return;
  if (flags && !flags[q]) return;  // second pass behind the tensor-core kernel: only the queries it could not serve
  const T* f1 = fmap1 + (size_t)q * C;
  for (int c = lane; c < C; c += 32) qv[c] = to_f32(f1[c]);
  __syncwarp();
  const float cx = coords[2 * (size_t)q], cy = coords[2 * (size_t)q + 1];
  const size_t b = (size_t)q / hw;
  const int planes = levels * K * K;
  for (int l = 0; l < levels; ++l) {
    const float s = 1.0f / (float)(1 << l);
    const float x = cx * s, y = cy * s;
    const int Hl = lv.h[l], Wl = lv.w[l];
    const bool finite = (fabsf(x) < 1e7f) && (fabsf(y) < 1e7f);
    const float xf = finite ? floorf(x) : -1e6f, yf = finite ? floorf(y) : -1e6f;
    const float fx = finite ? x - xf : 0.f, fy = finite ? y - yf : 0.f;
    const int x0 = (int)xf - r, y0 = (int)yf - r;
    const T* base = reinterpret_cast<const T*>(lv.ptr[l]) + b * (size_t)Hl * Wl * C;
    for (int t = lane; t < D * D; t += 32) {
      int j = t / D, i = t - j * D;
      int xi = x0 + i, yi = y0 + j;
      float v = 0.f;
      if (xi >= 0 && xi < Wl && yi >= 0 && yi < Hl) v = dot_row<T>(base + ((size_t)yi * Wl + xi) * C, qv, C);
      win[i * D + j] = v;
    }
    __syncwarp();
    const float w00 = (1.f - fx) * (1.f - fy) * scale, w10 = fx * (1.f - fy) * scale,
                w01 = (1.f - fx) * fy * scale, w11 = fx * fy * scale;
    for (int o = lane; o < K * K; o += 32) {
      int i = o / K, j = o - i * K;
      float v = w00 * win[i * D + j] + w10 * win[(i + 1) * D + j] + w01 * win[i * D + j + 1] +
                w11 * win[(i + 1) * D + j + 1];
      store_lookup<TO>(out, nchw, (size_t)q, hw, planes, out_stride, l * K * K + o, v);
    }
    __syncwarp();
  }
  // pixel-major output wider than the lookup: zero the pad columns (they meet zero weight rows)
  if (!nchw)
    for (int c = planes + lane; c < out_stride; c += 32) out[(size_t)q * out_stride + c] = from_f32<TO>(0.f);
}

// ------------------------------------------------------------------------------------------
static int fill_levels(LevelTable& lv, void* const* ptrs, int H, int W, int levels, const int* level_h = nullptr,
                       const int* level_w = nullptr) {
  for (int l = 0; l < levels; ++l) {
    if (!ptrs[l]) return -1;
    lv.ptr[l] = ptrs[l];
    lv.h[l] = level_h ? level_h[l] : H >> l;
    lv.w[l] = level_w ? level_w[l] : W >> l;
    if (lv.h[l] < 1 || lv.w[l] < 1) return -2;
  }
  return 0;
}

template <typename T>
static int launch_pool(const void* in, void* out, size_t N, int H, int W, int C, cudaStream_t s) {
  size_t total = N * (size_t)(H / 2) * (W / 2) * C;
  if (total == 0) return PFB_OK;
  int threads = 256;
  size_t blocks = ceil_div_sz(total, threads);
  size_t cap = (size_t)sm_count() * 32;
  if (blocks > cap) blocks = cap;
  ProfScope prof(KC_POOL, s);
  avg_pool2x2_kernel<T><<<(unsigned)blocks, threads, 0, s>>>(reinterpret_cast<const T*>(in),
                                                             reinterpret_cast<T*>(out), total, H, W, C);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

int corr_volume_simt(const void* f1, const void* f2, void* const* pyr, int B, int N1, int H, int W, int C, int L, float scale,
                     pfb_dtype dt, cudaStream_t s) {
  const int N2 = H * W;
  dim3 grid(ceil_div(N2, 64), ceil_div(N1, 64), B);
  PFB_DISPATCH_DTYPE(dt, T, {
    { ProfScope prof(KC_VOLUME, s);
    corr_volume_simt_kernel<T><<<grid, 256, 0, s>>>(reinterpret_cast<const T*>(f1),
                                                    reinterpret_cast<const T*>(f2),
                                                    reinterpret_cast<T*>(pyr[0]), N1, N2, C, scale); }
    PFB_LAUNCH_CHECK();
    for (int l = 1; l < L; ++l) {
      int rc = launch_pool<T>(pyr[l - 1], pyr[l], (size_t)B * N1, H >> (l - 1), W >> (l - 1), 1, s);
      if (rc) return rc;
    }
  });
  return PFB_OK;
}

int corr_onthefly_simt_flagged(const void* fmap1, void* const* pyr, const float* coords, void* out, const unsigned char* flags, int B, int H,
                               int W, int C, int levels, int radius, pfb_dtype dtype, int out_stride, cudaStream_t s, float scale);

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API size_t pfb_corr_level_bytes(int B, int H, int W, int level, pfb_dtype dtype) {
  return (size_t)B * H * W * (size_t)(H >> level) * (size_t)(W >> level) * dtype_size(dtype);
}

extern "C" PFB_API int pfb_corr_volume_build(const void* fmap1, const void* fmap2, void* const* pyramid, int B, int H,
                                     int W, int C, int levels, pfb_dtype dtype, int impl, pfb_stream stream) {
  return pfb_corr_volume_build_ex(fmap1, fmap2, pyramid, B, H, W, H, W, C, levels, 1.0f / sqrtf((float)(C > 0 ? C : 1)), dtype, impl,
                                  stream);
}

extern "C" PFB_API int pfb_corr_volume_build_ex(const void* fmap1, const void* fmap2, void* const* pyramid, int B, int H1, int W1,
                                                int H, int W, int C, int levels, float scale, pfb_dtype dtype, int impl,
                                                pfb_stream stream) {
  PFB_CHECK_ARG(fmap1 && fmap2 && pyramid, "corr_volume_build: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "corr_volume_build: bad dtype %d", (int)dtype);
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && H1 > 0 && W1 > 0 && C > 0, "corr_volume_build: bad shape B=%d queries %dx%d targets %dx%d C=%d", B,
                H1, W1, H, W, C);
  const int N1 = H1 * W1;
  PFB_CHECK_ARG(levels >= 1 && levels <= PFB_MAX_LEVELS, "corr_volume_build: levels=%d out of range", levels);
  PFB_CHECK_ARG((H >> (levels - 1)) >= 1 && (W >> (levels - 1)) >= 1,
                "corr_volume_build: %dx%d grid too small for %d levels", H, W, levels);
  for (int l = 0; l < levels; ++l) PFB_CHECK_ARG(pyramid[l], "corr_volume_build: pyramid[%d] is null", l);
  cudaStream_t s = as_stream(stream);
  bool can_umma = corr_volume_umma_supported(B, H, W, C, levels, dtype);
  if (impl == 2 && !can_umma) {
    set_error("corr_volume_build: wgmma path does not support B=%d H=%d W=%d C=%d dtype=%d", B, H, W, C, (int)dtype);
    return PFB_ERR_UNSUPPORTED;
  }
  if ((impl == 0 && can_umma) || impl == 2) return corr_volume_umma(fmap1, fmap2, pyramid, B, N1, H, W, C, levels, scale, dtype, s);
  return corr_volume_simt(fmap1, fmap2, pyramid, B, N1, H, W, C, levels, scale, dtype, s);
}

extern "C" PFB_API int pfb_avg_pool2x2_nhwc(const void* in, void* out, int N, int H, int W, int C, pfb_dtype dtype,
                                    pfb_stream stream) {
  PFB_CHECK_ARG(in && out, "avg_pool2x2: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && N > 0 && H > 0 && W > 0 && C > 0, "avg_pool2x2: bad arguments");
  PFB_DISPATCH_DTYPE(dtype, T, { return launch_pool<T>(in, out, (size_t)N, H, W, C, as_stream(stream)); });
  return PFB_OK;
}

template <typename T>
static int launch_lookup_t(const LevelTable& lv, const float* coords, void* out, int nq, int hw, int levels,
                           int radius, pfb_dtype out_dtype, int nchw, int out_stride, cudaStream_t s) {
  const int D = 2 * radius + 2;
  const int warps = 4;
  size_t smem = (size_t)warps * D * D * sizeof(float);
  dim3 grid(ceil_div(nq, warps));
  ProfScope prof(KC_LOOKUP, s);
  if (!nchw && (radius == 4 || radius == 3) && levels <= 4) {
#define PFB_LOOKUP_FAST(TO, R) launch_pdl(corr_lookup_r4_kernel<T, TO, R>, dim3(grid), dim3(128), 0, s, lv, coords, (TO*)out, nq, levels, out_stride)
    if (radius == 4) {
      if (out_dtype == PFB_F32) PFB_LOOKUP_FAST(float, 4);
      else if (out_dtype == PFB_F16) PFB_LOOKUP_FAST(__half, 4);
      else PFB_LOOKUP_FAST(__nv_bfloat16, 4);
    } else {
      if (out_dtype == PFB_F32) PFB_LOOKUP_FAST(float, 3);
      else if (out_dtype == PFB_F16) PFB_LOOKUP_FAST(__half, 3);
      else PFB_LOOKUP_FAST(__nv_bfloat16, 3);
    }
#undef PFB_LOOKUP_FAST
    PFB_LAUNCH_CHECK();
    return PFB_OK;
  }
  if (out_dtype == PFB_F32)
    corr_lookup_kernel<T, float><<<grid, warps * 32, smem, s>>>(lv, coords, (float*)out, nq, hw, levels, radius, nchw, out_stride);
  else if (out_dtype == PFB_F16)
    corr_lookup_kernel<T, __half><<<grid, warps * 32, smem, s>>>(lv, coords, (__half*)out, nq, hw, levels, radius, nchw, out_stride);
  else
    corr_lookup_kernel<T, __nv_bfloat16><<<grid, warps * 32, smem, s>>>(lv, coords, (__nv_bfloat16*)out, nq, hw, levels, radius, nchw, out_stride);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_corr_level_sizes(int H, int W, int levels, int pool_min_side, int* level_h, int* level_w) {
  PFB_CHECK_ARG(level_h && level_w, "corr_level_sizes: null output");
  PFB_CHECK_ARG(H > 0 && W > 0, "corr_level_sizes: bad grid %dx%d", H, W);
  PFB_CHECK_ARG(levels >= 1 && levels <= PFB_MAX_LEVELS, "corr_level_sizes: levels=%d out of range", levels);
  PFB_CHECK_ARG(pool_min_side >= 0, "corr_level_sizes: pool_min_side=%d", pool_min_side);
  int distinct = 1;
  level_h[0] = H;
  level_w[0] = W;
  for (int l = 1; l < levels; ++l) {
    const int ph = level_h[l - 1], pw = level_w[l - 1];
    const bool pool = pool_min_side == 0 || (ph < pw ? ph : pw) > pool_min_side;
    level_h[l] = pool ? ph / 2 : ph;
    level_w[l] = pool ? pw / 2 : pw;
    distinct += pool;
  }
  return distinct;
}

extern "C" PFB_API int pfb_corr_lookup(void* const* pyramid, const float* coords, void* out, int B, int H, int W,
                               int levels, int radius, pfb_dtype dtype, pfb_dtype out_dtype, int out_nchw,
                               int out_stride, pfb_stream stream) {
  return pfb_corr_lookup_ex(pyramid, nullptr, nullptr, coords, out, B, H, W, levels, radius, dtype, out_dtype, out_nchw, out_stride,
                            stream);
}

extern "C" PFB_API int pfb_corr_lookup_ex(void* const* pyramid, const int* level_h, const int* level_w, const float* coords, void* out,
                                          int B, int H, int W, int levels, int radius, pfb_dtype dtype, pfb_dtype out_dtype,
                                          int out_nchw, int out_stride, pfb_stream stream) {
  PFB_CHECK_ARG(pyramid && coords && out, "corr_lookup: null pointer");
  PFB_CHECK_ARG((level_h == nullptr) == (level_w == nullptr), "corr_lookup: level_h and level_w come together");
  PFB_CHECK_ARG(dtype_ok(dtype) && dtype_ok(out_dtype), "corr_lookup: bad dtype");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0, "corr_lookup: bad shape");
  PFB_CHECK_ARG(levels >= 1 && levels <= PFB_MAX_LEVELS, "corr_lookup: levels=%d out of range", levels);
  PFB_CHECK_ARG(radius >= 0 && radius <= 15, "corr_lookup: radius=%d out of range", radius);
  const int planes = levels * (2 * radius + 1) * (2 * radius + 1);
  PFB_CHECK_ARG(out_nchw || out_stride >= planes, "corr_lookup: out_stride=%d < %d planes", out_stride, planes);
  LevelTable lv;
  int rc = fill_levels(lv, pyramid, H, W, levels, level_h, level_w);
  PFB_CHECK_ARG(rc == 0, "corr_lookup: pyramid level missing or empty (rc=%d)", rc);
  PFB_DISPATCH_DTYPE(dtype, T, {
    return launch_lookup_t<T>(lv, coords, out, B * H * W, H * W, levels, radius, out_dtype, out_nchw, out_stride,
                              as_stream(stream));
  });
  return PFB_OK;
}

template <typename T>
static int launch_onthefly_t(const void* fmap1, const LevelTable& lv, const float* coords, void* out, int nq,
                             int hw, int C, int levels, int radius, float scale, pfb_dtype out_dtype, int nchw,
                             int out_stride, cudaStream_t s, const unsigned char* flags = nullptr) {
  const int D = 2 * radius + 2;
  const int warps = 4;
  size_t smem = (size_t)warps * (C + D * D) * sizeof(float);
  dim3 grid(ceil_div(nq, warps));
  const T* f1 = reinterpret_cast<const T*>(fmap1);
  ProfScope prof(KC_ONTHEFLY, s);
#define PFB_OTF(TO)                                                                                         \
  do {                                                                                                      \
    if (smem > 48 * 1024)                                                                                   \
      PFB_CUDA(cudaFuncSetAttribute(corr_onthefly_kernel<T, TO>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    corr_onthefly_kernel<T, TO><<<grid, warps * 32, smem, s>>>(f1, lv, coords, (TO*)out, nq, hw, C, levels,  \
                                                               radius, scale, nchw, out_stride, flags);     \
  } while (0)
  if (out_dtype == PFB_F32) PFB_OTF(float);
  else if (out_dtype == PFB_F16) PFB_OTF(__half);
  else PFB_OTF(__nv_bfloat16);
#undef PFB_OTF
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_corr_lookup_onthefly(const void* fmap1, void* const* fmap2_pyramid, const float* coords,
                                        void* out, int B, int H, int W, int C, int levels, int radius,
                                        pfb_dtype dtype, pfb_dtype out_dtype, int out_nchw, int out_stride,
                                        pfb_stream stream) {
  return pfb_corr_lookup_onthefly_ex(fmap1, fmap2_pyramid, coords, out, B, H, W, C, levels, radius, 0.f, dtype, out_dtype, out_nchw,
                                     out_stride, stream);
}

extern "C" PFB_API int pfb_corr_lookup_onthefly_ex(const void* fmap1, void* const* fmap2_pyramid, const float* coords, void* out, int B,
                                                   int H, int W, int C, int levels, int radius, float scale, pfb_dtype dtype,
                                                   pfb_dtype out_dtype, int out_nchw, int out_stride, pfb_stream stream) {
  PFB_CHECK_ARG(fmap1 && fmap2_pyramid && coords && out, "corr_lookup_onthefly: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && dtype_ok(out_dtype), "corr_lookup_onthefly: bad dtype");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "corr_lookup_onthefly: C=%d must be a positive multiple of 8", C);
  PFB_CHECK_ARG(levels >= 1 && levels <= PFB_MAX_LEVELS, "corr_lookup_onthefly: levels=%d out of range", levels);
  PFB_CHECK_ARG(radius >= 0 && radius <= 15, "corr_lookup_onthefly: radius=%d out of range", radius);
  const int planes = levels * (2 * radius + 1) * (2 * radius + 1);
  PFB_CHECK_ARG(out_nchw || out_stride >= planes, "corr_lookup_onthefly: out_stride=%d < %d planes", out_stride, planes);
  LevelTable lv;
  int rc = fill_levels(lv, fmap2_pyramid, H, W, levels);
  PFB_CHECK_ARG(rc == 0, "corr_lookup_onthefly: fmap2 level missing or empty (rc=%d)", rc);
  PFB_CHECK_ARG(scale >= 0.f, "corr_lookup_onthefly: scale=%g", (double)scale);
  if (scale == 0.f) scale = 1.0f / sqrtf((float)C);
  PFB_DISPATCH_DTYPE(dtype, T, {
    return launch_onthefly_t<T>(fmap1, lv, coords, out, B * H * W, H * W, C, levels, radius, scale, out_dtype,
                                out_nchw, out_stride, as_stream(stream));
  });
  return PFB_OK;
}

extern "C" PFB_API int pfb_alt_corr_forward(const void* fmap1, const void* fmap2, const float* coords, void* out, int B,
                                    int H1, int W1, int H2, int W2, int C, int radius, pfb_dtype dtype,
                                    pfb_dtype out_dtype, pfb_stream stream) {
  PFB_CHECK_ARG(fmap1 && fmap2 && coords && out, "alt_corr_forward: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && dtype_ok(out_dtype), "alt_corr_forward: bad dtype");
  PFB_CHECK_ARG(B > 0 && H1 > 0 && W1 > 0 && H2 > 0 && W2 > 0 && C > 0 && C % 8 == 0,
                "alt_corr_forward: bad shape (C=%d must be a multiple of 8)", C);
  PFB_CHECK_ARG(radius >= 0 && radius <= 15, "alt_corr_forward: radius=%d out of range", radius);
  LevelTable lv;
  lv.ptr[0] = fmap2;
  lv.h[0] = H2;
  lv.w[0] = W2;
  PFB_DISPATCH_DTYPE(dtype, T, {
    return launch_onthefly_t<T>(fmap1, lv, coords, out, B * H1 * W1, H1 * W1, C, 1, radius, 1.0f, out_dtype,
                                /*nchw=*/1, 0, as_stream(stream));
  });
  return PFB_OK;
}

namespace pfb {
int corr_onthefly_simt_flagged(const void* fmap1, void* const* pyr, const float* coords, void* out, const unsigned char* flags, int B, int H,
                               int W, int C, int levels, int radius, pfb_dtype dtype, int out_stride, cudaStream_t s, float scale) {
  LevelTable lv;
  if (fill_levels(lv, pyr, H, W, levels) != 0) {
    set_error("corr_onthefly (flagged pass): fmap2 level missing or empty");
    return PFB_ERR_ARG;
  }
  if (scale == 0.f) scale = 1.0f / sqrtf((float)C);
  PFB_DISPATCH_DTYPE(dtype, T, {
    return launch_onthefly_t<T>(fmap1, lv, coords, out, B * H * W, H * W, C, levels, radius, scale, dtype, 0, out_stride, s, flags);
  });
  return PFB_OK;
}
}  // namespace pfb
