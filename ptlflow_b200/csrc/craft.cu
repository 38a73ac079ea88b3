// CRAFT (a23): the batch-global clamp flag, the windowed-bias attention softmax, the mode soft-aggregate with skip and LayerNorm,
// and the inter-frame volume's mode mix with its global LayerNorm.  See include/ptlflow_b200.h, a23.
#include <atomic>

#include "common.cuh"
#include "corr_umma.cuh"
#include "softmax_row.cuh"

namespace pfb {

namespace {

constexpr int kMaxModes = 4;
constexpr int kMaxBiasRadius = 15;
constexpr float kLnEps = 1e-12f;
constexpr int kStatBlocks = 512;  // CTAs per sample of the volume mix (fixed: the statistics' summation order depends on it)
constexpr int kStatThreads = 256;

// ---- the clamp flag: *flag = any(x > clip).  The caller zeroes the flag first; every writer stores the same 1. ----
template <typename T>
__global__ void clamp_flag_kernel(const T* __restrict__ x, size_t n, float clip, int* __restrict__ flag) {
  bool hit = false;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) hit |= to_f32(x[i]) > clip;
  if (__syncthreads_or(hit) && threadIdx.x == 0) *flag = 1;
}

// the weighted window bias of the key (ky, kx) for the query (qy, qx); 0 outside the (2R+1)^2 window
__device__ __forceinline__ float window_bias(const float* bias, int R, int dy, int dx) {
  return (abs(dy) <= R && abs(dx) <= R) ? bias[(dy + R) * (2 * R + 1) + (dx + R)] : 0.f;
}

// ---- windowed-bias softmax: one CTA per row r (query i = r % N), in place ----
template <typename T, bool VEC>
__global__ void __launch_bounds__(kRowThreads) window_softmax_kernel(T* logits, const float* __restrict__ bias_tab, int H, int W, int R,
                                                                     int mask_radius, const int* __restrict__ flag, float clip) {
  extern __shared__ __align__(16) float srow[];  // [N] row, then the (2R+1)^2 bias table
  __shared__ float red[kRowThreads / 32];
  const int N = H * W, K = 2 * R + 1;
  float* bias = srow + ((N + 3) & ~3);
  for (int t = threadIdx.x; t < K * K; t += kRowThreads) bias[t] = bias_tab[t];
  __syncthreads();
  const size_t r = blockIdx.x;
  const int i = (int)(r % (size_t)N), qy = i / W, qx = i - qy * W;
  const bool clamp = *flag != 0;
  T* row = logits + r * N;
  softmax_row_smem<T, VEC>(row, row, N, W, srow, red, [&](float f, int ky, int kx) {
    if (clamp) f = fminf(fmaxf(f, -clip), clip);
    const int dy = ky - qy, dx = kx - qx;
    f += window_bias(bias, R, dy, dx);
    if (mask_radius > 0 && max(abs(dy), abs(dx)) > mask_radius) f += -1e9f;
    return f;
  });
}

// ---- mode soft-aggregate + skip + LayerNorm: one warp per pixel, F / 32 channels per lane (lane-interleaved) ----
template <typename T, int F>
__global__ void mode_aggregate_kernel(const T* feat, int feat_stride, int M, const float* __restrict__ w, float coeff, const T* skip,
                                      int skip_stride, T* out, int out_stride, int P) {
  constexpr int CPL = F / 32;
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (p >= P) return;
  float y[kMaxModes][CPL], score[kMaxModes];
  const T* fp = feat + (size_t)p * feat_stride;
#pragma unroll
  for (int m = 0; m < kMaxModes; ++m) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < CPL; ++k) {
      y[m][k] = m < M ? to_f32(fp[m * F + k * 32 + lane]) : 0.f;
      s += w[k * 32 + lane] * y[m][k];
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    score[m] = s;
  }
  float mx = score[0];
#pragma unroll
  for (int m = 1; m < kMaxModes; ++m)
    if (m < M) mx = fmaxf(mx, score[m]);
  float pi[kMaxModes], den = 0.f;
#pragma unroll
  for (int m = 0; m < kMaxModes; ++m) {
    pi[m] = m < M ? expf(score[m] - mx) : 0.f;
    den += pi[m];
  }
  const T* sp = skip + (size_t)p * skip_stride;
  float t[CPL], sum = 0.f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) {
    float a = 0.f;
#pragma unroll
    for (int m = 0; m < kMaxModes; ++m) a += pi[m] * y[m][k];
    t[k] = coeff * to_f32(sp[k * 32 + lane]) + a / den;
    sum += t[k];
  }
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / F;
  float var = 0.f;
#pragma unroll
  for (int k = 0; k < CPL; ++k) var += (t[k] - mean) * (t[k] - mean);
  for (int o = 16; o > 0; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  const float rstd = rsqrtf(var / F + kLnEps);
  T* op = out + (size_t)p * out_stride;
  __syncwarp();  // out may alias feat (one mode, in place): every lane has read its inputs
#pragma unroll
  for (int k = 0; k < CPL; ++k) op[k * 32 + lane] = from_f32<T>((t[k] - mean) * rstd);
}

// ---- inter-frame volume: mode mix of the clamped, biased scores into fp32, with per-CTA fp64 partial sums ----
template <typename T>
__global__ void __launch_bounds__(kStatThreads) volume_mix_kernel(const T* __restrict__ scores, int M, int B, int H, int W, float a,
                                                                  const float* __restrict__ bias_tab, int R, const int* __restrict__ flag,
                                                                  float clip, float* __restrict__ mix, double* __restrict__ partial) {
  __shared__ float bias[(2 * kMaxBiasRadius + 1) * (2 * kMaxBiasRadius + 1)];
  __shared__ double red[2][kStatThreads / 32];
  const int K = 2 * R + 1;
  for (int t = threadIdx.x; t < K * K; t += kStatThreads) bias[t] = bias_tab[t];
  __syncthreads();
  const int b = blockIdx.y, N = H * W;
  const size_t NN = (size_t)N * N;
  const bool clamp = *flag != 0;
  double s1 = 0.0, s2 = 0.0;
  for (size_t e = blockIdx.x * (size_t)kStatThreads + threadIdx.x; e < NN; e += (size_t)gridDim.x * kStatThreads) {
    const int i = (int)(e / N), j = (int)(e - (size_t)i * N);
    const int qy = i / W, qx = i - qy * W, ky = j / W, kx = j - ky * W;
    const float pb = window_bias(bias, R, ky - qy, kx - qx);
    float s[kMaxModes], mx = -INFINITY;
#pragma unroll
    for (int m = 0; m < kMaxModes; ++m) {
      if (m >= M) break;
      float v = to_f32(scores[((size_t)m * B + b) * NN + e]);
      if (clamp) v = fminf(fmaxf(v, -clip), clip);
      s[m] = v + pb;
      mx = fmaxf(mx, a * s[m]);
    }
    float v = s[0];
    if (M > 1) {  // sum_m softmax_m(a s_m + c) s_m: the feat2score bias c cancels
      float num = 0.f, den = 0.f;
#pragma unroll
      for (int m = 0; m < kMaxModes; ++m) {
        if (m >= M) break;
        const float p = expf(a * s[m] - mx);
        num += p * s[m];
        den += p;
      }
      v = num / den;
    }
    mix[(size_t)b * NN + e] = v;
    s1 += v;
    s2 += (double)v * v;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (lane == 0) { red[0][warp] = s1; red[1][warp] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t1 = 0.0, t2 = 0.0;
    for (int w = 0; w < kStatThreads / 32; ++w) { t1 += red[0][w]; t2 += red[1][w]; }
    partial[((size_t)b * gridDim.x + blockIdx.x) * 2] = t1;
    partial[((size_t)b * gridDim.x + blockIdx.x) * 2 + 1] = t2;
  }
}

// the partial sums of one sample in a fixed order -> (mean, rstd) fp32; one CTA of 32 threads per sample
__global__ void volume_stats_kernel(const double* __restrict__ partial, int nblk, size_t n, float* __restrict__ stats) {
  const int b = blockIdx.x, lane = threadIdx.x;
  double s1 = 0.0, s2 = 0.0;
  for (int k = lane; k < nblk; k += 32) {
    s1 += partial[((size_t)b * nblk + k) * 2];
    s2 += partial[((size_t)b * nblk + k) * 2 + 1];
  }
  for (int o = 16; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (lane == 0) {
    const double mean = s1 / (double)n, var = fmax(s2 / (double)n - mean * mean, 0.0);
    stats[2 * b] = (float)mean;
    stats[2 * b + 1] = (float)(1.0 / sqrt(var + (double)kLnEps));
  }
}

template <typename T>
__global__ void volume_normalize_kernel(const float* __restrict__ mix, const float* __restrict__ stats, size_t NN, T* __restrict__ out) {
  const int b = blockIdx.y;
  const float mean = stats[2 * b], rstd = stats[2 * b + 1];
  for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < NN; e += (size_t)gridDim.x * blockDim.x)
    out[(size_t)b * NN + e] = from_f32<T>((mix[(size_t)b * NN + e] - mean) * rstd);
}

template <typename T, bool VEC>
int launch_window_softmax(void* logits, size_t rows, int H, int W, const float* bias, int R, int mask_radius, const int* flag, float clip,
                          cudaStream_t s) {
  const size_t smem = (size_t)(((H * W + 3) & ~3) + (2 * R + 1) * (2 * R + 1)) * sizeof(float);
  static std::atomic<unsigned long long> attr_done{0};  // once per (instantiation, device)
  int dev = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  if (!(attr_done.load(std::memory_order_acquire) & (1ull << (dev & 63)))) {
    PFB_CUDA(cudaFuncSetAttribute(window_softmax_kernel<T, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
  }
  window_softmax_kernel<T, VEC><<<(unsigned)rows, kRowThreads, smem, s>>>((T*)logits, bias, H, W, R, mask_radius, flag, clip);
  return PFB_OK;
}


// ---- the fused inter-frame volume on wgmma (f16 / bf16), three passes over the same K = 256 GEMM ----
//
// CTA = 13 warps as shift_volume_tiled_kernel: 0-3 epilogue (thread = query row), 4-11 two MMA warpgroups (64 query rows each),
// 12 TMA producer.  One work item per CTA: 128 queries x one 16 x 8 target patch.  The four 64-channel K chunks of q1 and k2 arrive
// at once (no ring: 128 KB).  Mode m owns chunks [m * 4 / M, (m + 1) * 4 / M).  Each MMA warpgroup runs the patch as four 32-column
// quarters (m64n32): per quarter and mode it accumulates the mode's chunks, then folds the score into the online mode mix, held as a
// log-sum-exp L = log sum_m exp(a s_m) and the running mix v (two fp32 values beside each accumulator, 48 registers in all; with
// m64n64 halves the 96 spilled under the 13-warp CTA's register budget):
//   s = (flag ? clamp(d scale) : d scale) + bias,   L' = logaddexp(L, a s),   v' = v + exp(a s - L') (s - v).
//   PASS 0: any raw score above clip over the whole call -> *flag (the caller zeroes it).
//   PASS 1: per-CTA fp64 sums of v and v^2 over the patch's in-map elements -> partial[b][cta][2] (fixed order).
//   PASS 2: (v - mean_b) rstd_b into the accumulator tile, written by tiled_epilogue_item (levels 0-3 of the tiled pyramid).
constexpr int kCraftChunks = 4;  // K = 256

struct __align__(8) CraftBars {
  uint64_t full[kCraftChunks];
  uint64_t acc_full;
  uint64_t acc_empty;
};

template <typename T, int PASS>
__global__ void __launch_bounds__(kCorrThreads, 1)
craft_volume_tiled_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                          const __grid_constant__ CUtensorMap tmO, TiledOut out, int H, int W, int N1, int M, float scale, float a,
                          const float* __restrict__ bias_tab, int R, int* __restrict__ flag, float clip, double* __restrict__ partial,
                          const float* __restrict__ stats, int levels) {
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sStage = smem;                                                           // 4 x (A 16 KB | B 16 KB)
  float* sacc = reinterpret_cast<float*>(sStage + kCraftChunks * 2 * kTileBytes);  // fp32 accumulator tile, 128 columns
  uint8_t* sC = sStage;  // level-0 staging (32 KB): the operand stages are free once the accumulators are handed over
  CraftBars* bars = reinterpret_cast<CraftBars*>(reinterpret_cast<uint8_t*>(sacc) + acc_tile_bytes(128));
  __shared__ double red[2][kCorrThreads / 32];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int PW = (W + 15) / 16;
  const int ph = blockIdx.x / PW, pw = blockIdx.x - ph * PW;
  const int m_tile = blockIdx.y, b = blockIdx.z;

  if (threadIdx.x == 0) {
    for (int k = 0; k < kCraftChunks; ++k) mbar_init(&bars->full[k], 1);
    mbar_init(&bars->acc_full, 8);
    mbar_init(&bars->acc_empty, 4);
    fence_barrier_init();
  }
  if (warp == 12 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (PASS == 2) prefetch_tmap(&tmO);
  }
  __syncthreads();

  bool hit = false;
  float s1 = 0.f, s2 = 0.f;
  if (warp == 12) {
    // ================= TMA producer =================
    if (lane == 0) {
      for (int k = 0; k < kCraftChunks; ++k) {
        uint8_t* sa = sStage + k * 2 * kTileBytes;
        mbar_arrive_expect_tx(&bars->full[k], 2 * kTileBytes);
        tma_load_3d(sa, &tmA, &bars->full[k], k * 64, m_tile * 128, b);
        tma_load_4d(sa + kTileBytes, &tmB, &bars->full[k], k * 64, pw * 16, ph * 8, b);
      }
    }
  } else if (warp >= 4) {
    // ================= MMA warpgroups =================
    const int wg = (threadIdx.x >> 7) - 1, tid = threadIdx.x & 127;
    const int kpm = kCraftChunks / M;
    const bool clamp = PASS > 0 && *flag != 0;
    const int K = 2 * R + 1;
    float mean = 0.f, rstd = 1.f;
    if (PASS == 2) { mean = stats[2 * b]; rstd = stats[2 * b + 1]; }
    for (int k = 0; k < kCraftChunks; ++k) mbar_wait(&bars->full[k], 0);
#pragma unroll 1
    for (int h = 0; h < 4; ++h) {
      float d[16], L[16], v[16];
#pragma unroll 1
      for (int m = 0; m < M; ++m) {
        wgmma_fence();
#pragma unroll 1
        for (int k = m * kpm; k < (m + 1) * kpm; ++k) {
          const uint32_t sa = smem_u32(sStage + k * 2 * kTileBytes);
          const uint32_t al = gdesc_lo(sa + wg * 64 * 128, 16), bl = gdesc_lo(sa + kTileBytes + h * 32 * 128, 16);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            wgmma<32, BF16>(d, gdesc(al + 2 * kk, kDescHiSw128), gdesc(bl + 2 * kk, kDescHiSw128), (k == m * kpm && kk == 0) ? 0u : 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(d);
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const int n1 = m_tile * 128 + wg * 64 + frag_row(tid, e);
          const int col = h * 32 + frag_col(tid, e), y = ph * 8 + (col >> 4), x = pw * 16 + (col & 15);
          const bool valid = n1 < N1 && y < H && x < W;
          const float raw = d[e] * scale;
          if (PASS == 0) {
            hit |= valid && raw > clip;
            continue;
          }
          const int qy = n1 / W, qx = n1 - qy * W, dy = y - qy, dx = x - qx;
          float sv = clamp ? fminf(fmaxf(raw, -clip), clip) : raw;
          if (abs(dy) <= R && abs(dx) <= R) sv += __ldg(bias_tab + (dy + R) * K + (dx + R));
          if (m == 0) {
            L[e] = a * sv;
            v[e] = sv;
          } else {
            const float as = a * sv, mx = fmaxf(L[e], as);
            const float Ln = mx + log1pf(__expf(-fabsf(L[e] - as)));
            v[e] += __expf(as - Ln) * (sv - v[e]);
            L[e] = Ln;
          }
        }
      }
      if (PASS == 1) {
#pragma unroll
        for (int e = 0; e < 16; ++e) {
          const int n1 = m_tile * 128 + wg * 64 + frag_row(tid, e);
          const int col = h * 32 + frag_col(tid, e), y = ph * 8 + (col >> 4), x = pw * 16 + (col & 15);
          if (n1 < N1 && y < H && x < W) { s1 += v[e]; s2 += v[e] * v[e]; }
        }
      } else if (PASS == 2) {
#pragma unroll
        for (int e = 0; e < 16; ++e) v[e] = (v[e] - mean) * rstd;
        acc_store<32>(sacc + h * 32 * kAccPitch, v, wg * 64, tid);
      }
    }
    if (PASS == 2) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->acc_full);
    }
  } else if (PASS == 2) {
    // ================= epilogue: 4 warps, thread <-> query row =================
    const int row = (warp & 3) * 32 + lane;
    const int n1 = m_tile * 128 + row;
    const bool row_ok = n1 < N1;
    const size_t q = (size_t)b * N1 + (row_ok ? n1 : 0);
    T* o1 = levels > 1 ? reinterpret_cast<T*>(out.ptr[1]) + q * out.map_elems[1] : nullptr;
    T* o2 = levels > 2 ? reinterpret_cast<T*>(out.ptr[2]) + q * out.map_elems[2] : nullptr;
    T* o3 = levels > 3 ? reinterpret_cast<T*>(out.ptr[3]) + q * out.map_elems[3] : nullptr;
    tiled_epilogue_item<T>(sacc, sC, &tmO, out, row, row_ok, o1, o2, o3, 0, ph, pw, m_tile, b, 1.0f, &bars->acc_full, &bars->acc_empty);
    if (row == 0) tma_store_wait_read();
  }
  if (PASS == 0) {
    if (__syncthreads_or(hit) && threadIdx.x == 0) *flag = 1;
  } else if (PASS == 1) {
    double t1 = s1, t2 = s2;
    for (int o = 16; o > 0; o >>= 1) {
      t1 += __shfl_xor_sync(0xffffffffu, t1, o);
      t2 += __shfl_xor_sync(0xffffffffu, t2, o);
    }
    if (lane == 0) { red[0][warp] = t1; red[1][warp] = t2; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double u1 = 0.0, u2 = 0.0;
      for (int w = 0; w < kCorrThreads / 32; ++w) { u1 += red[0][w]; u2 += red[1][w]; }
      const size_t cta = ((size_t)b * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
      partial[2 * cta] = u1;
      partial[2 * cta + 1] = u2;
    }
  }
}

template <typename T, int PASS>
static int launch_craft_tiled(dim3 grid, size_t smem, cudaStream_t s, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO,
                              const TiledOut& out, int H, int W, int N1, int M, float scale, float a, const float* bias, int R, int* flag,
                              float clip, double* partial, const float* stats, int levels) {
  PFB_CUDA(cudaFuncSetAttribute(craft_volume_tiled_kernel<T, PASS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  craft_volume_tiled_kernel<T, PASS><<<grid, kCorrThreads, smem, s>>>(tmA, tmB, tmO, out, H, W, N1, M, scale, a, bias, R, flag, clip, partial,
                                                                      stats, levels);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_craft_clamp_flag(const void* x, size_t n, float clip, int* flag, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && flag && n > 0 && dtype_ok(dtype), "craft_clamp_flag: null pointer, empty input or bad dtype");
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), s));
  const unsigned grid = (unsigned)std::min<size_t>(ceil_div_sz(n, 256), (size_t)sm_count() * 8);
  PFB_DISPATCH_DTYPE(dtype, T, { clamp_flag_kernel<T><<<grid, 256, 0, s>>>((const T*)x, n, clip, flag); });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_craft_window_softmax(void* logits, size_t rows, int H, int W, const float* bias, int R, int mask_radius,
                                                const int* flag, float clip, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(logits && bias && flag && dtype_ok(dtype), "craft_window_softmax: null pointer or bad dtype");
  PFB_CHECK_ARG(H > 0 && W > 0 && H <= 200 && W <= 200, "craft_window_softmax: %dx%d grid outside 1..200 per side", H, W);
  PFB_CHECK_ARG(R >= 0 && R <= kMaxBiasRadius, "craft_window_softmax: bias radius %d outside 0..%d", R, kMaxBiasRadius);
  const size_t N = (size_t)H * W;
  PFB_CHECK_ARG(rows > 0 && rows < (1ull << 31) && rows % N == 0, "craft_window_softmax: rows=%zu is not a multiple of H*W=%zu", rows, N);
  cudaStream_t s = as_stream(stream);
  const bool vec = N % (16 / dtype_size(dtype)) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0;
  int rc = PFB_OK;
  {
    ProfScope prof(KC_MISC, s);
    PFB_DISPATCH_DTYPE(dtype, T, {
      rc = vec ? launch_window_softmax<T, true>(logits, rows, H, W, bias, R, mask_radius, flag, clip, s)
               : launch_window_softmax<T, false>(logits, rows, H, W, bias, R, mask_radius, flag, clip, s);
    });
  }
  if (rc != PFB_OK) return rc;
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_craft_mode_aggregate(const void* feat, int feat_stride, int M, int F, const float* w, float coeff, const void* skip,
                                                int skip_stride, int skip_offset, void* out, int out_stride, int out_offset, int P,
                                                pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(feat && w && skip && out && dtype_ok(dtype), "craft_mode_aggregate: null pointer or bad dtype");
  PFB_CHECK_ARG(M >= 1 && M <= kMaxModes && (F == 128 || F == 256) && P > 0, "craft_mode_aggregate: M=%d F=%d P=%d", M, F, P);
  PFB_CHECK_ARG(feat_stride >= M * F && skip_offset >= 0 && skip_stride >= skip_offset + F && out_offset >= 0 && out_stride >= out_offset + F,
                "craft_mode_aggregate: strides / offsets do not hold %d x %d features", M, F);
  cudaStream_t s = as_stream(stream);
  const int warps = 8;
  const unsigned grid = (unsigned)ceil_div(P, warps);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    const T* sk = (const T*)skip + skip_offset;
    T* o = (T*)out + out_offset;
    if (F == 128) mode_aggregate_kernel<T, 128><<<grid, warps * 32, 0, s>>>((const T*)feat, feat_stride, M, w, coeff, sk, skip_stride, o, out_stride, P);
    else mode_aggregate_kernel<T, 256><<<grid, warps * 32, 0, s>>>((const T*)feat, feat_stride, M, w, coeff, sk, skip_stride, o, out_stride, P);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API size_t pfb_craft_volume_workspace_bytes(int B, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  const size_t NN = (size_t)H * W * H * W;
  return align_up((size_t)B * NN * sizeof(float), 256) + align_up((size_t)B * kStatBlocks * 2 * sizeof(double), 256) +
         align_up((size_t)B * 2 * sizeof(float), 256);
}

extern "C" PFB_API int pfb_craft_volume_norm(const void* scores, int M, float a, const float* bias, int R, const int* flag, float clip,
                                             void* level0, void* workspace, size_t workspace_bytes, int B, int H, int W, pfb_dtype dtype,
                                             pfb_stream stream) {
  PFB_CHECK_ARG(scores && bias && flag && level0 && workspace && dtype_ok(dtype), "craft_volume_norm: null pointer or bad dtype");
  PFB_CHECK_ARG(M >= 1 && M <= kMaxModes, "craft_volume_norm: %d modes outside 1..%d", M, kMaxModes);
  PFB_CHECK_ARG(R >= 0 && R <= kMaxBiasRadius, "craft_volume_norm: bias radius %d outside 0..%d", R, kMaxBiasRadius);
  PFB_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && W > 0, "craft_volume_norm: bad grid %dx%dx%d", B, H, W);
  const size_t need = pfb_craft_volume_workspace_bytes(B, H, W);
  PFB_CHECK_ARG(workspace_bytes >= need, "craft_volume_norm: workspace %zu bytes < required %zu", workspace_bytes, need);
  const size_t NN = (size_t)H * W * H * W;
  char* ws = reinterpret_cast<char*>(workspace);
  float* mix = reinterpret_cast<float*>(ws);
  double* partial = reinterpret_cast<double*>(ws + align_up((size_t)B * NN * sizeof(float), 256));
  float* stats = reinterpret_cast<float*>(ws + align_up((size_t)B * NN * sizeof(float), 256) + align_up((size_t)B * kStatBlocks * 2 * sizeof(double), 256));
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    volume_mix_kernel<T><<<dim3(kStatBlocks, B), kStatThreads, 0, s>>>((const T*)scores, M, B, H, W, a, bias, R, flag, clip, mix, partial);
    volume_stats_kernel<<<B, 32, 0, s>>>(partial, kStatBlocks, NN, stats);
    volume_normalize_kernel<T><<<dim3((unsigned)std::min<size_t>(ceil_div_sz(NN, 256), 4096), B), 256, 0, s>>>(mix, stats, NN, (T*)level0);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

static size_t craft_tiled_ctas(int B, int H, int W) { return (size_t)B * ceil_div(H * W, 128) * (ceil_div(W, 16) * ceil_div(H, 8)); }

extern "C" PFB_API size_t pfb_craft_volume_tiled_workspace_bytes(int B, int H, int W) {
  if (B <= 0 || H <= 0 || W <= 0) return 0;
  return align_up(craft_tiled_ctas(B, H, W) * 2 * sizeof(double), 256) + align_up((size_t)B * 2 * sizeof(float), 256) + 256;
}

extern "C" PFB_API int pfb_craft_volume_tiled(const void* q1, const void* k2, int M, float a, const float* bias, int R, int* flag, float clip,
                                              void* const* pyramid, void* workspace, size_t workspace_bytes, int B, int H, int W, int levels,
                                              pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(q1 && k2 && bias && flag && pyramid && workspace, "craft_volume_tiled: null pointer");
  PFB_CHECK_ARG(dtype == PFB_F16 || dtype == PFB_BF16, "craft_volume_tiled: f16 / bf16 only (dtype=%d)", (int)dtype);
  PFB_CHECK_ARG(M == 1 || M == 2 || M == 4, "craft_volume_tiled: %d modes (1, 2 or 4: modes of 64-channel multiples)", M);
  PFB_CHECK_ARG(R >= 0 && R <= kMaxBiasRadius, "craft_volume_tiled: bias radius %d outside 0..%d", R, kMaxBiasRadius);
  PFB_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && W > 0, "craft_volume_tiled: bad grid %dx%dx%d", B, H, W);
  PFB_CHECK_ARG(levels >= 1 && levels <= 4 && (H >> (levels - 1)) >= 1 && (W >> (levels - 1)) >= 1,
                "craft_volume_tiled: %dx%d grid cannot hold %d levels (1..4)", H, W, levels);
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(q1) & 15) == 0 && (reinterpret_cast<uintptr_t>(k2) & 15) == 0,
                "craft_volume_tiled: operands must be 16-byte aligned");
  for (int l = 0; l < levels; ++l)
    PFB_CHECK_ARG(pyramid[l] && (reinterpret_cast<uintptr_t>(pyramid[l]) & 15) == 0, "craft_volume_tiled: pyramid[%d] null or not 16-byte aligned", l);
  const size_t need = pfb_craft_volume_tiled_workspace_bytes(B, H, W);
  PFB_CHECK_ARG(workspace_bytes >= need, "craft_volume_tiled: workspace %zu bytes < required %zu", workspace_bytes, need);
  const int N1 = H * W, C = 256;
  const int m_tiles = ceil_div(N1, 128), n_patches = ceil_div(W, 16) * ceil_div(H, 8);
  PFB_CHECK_ARG(m_tiles <= 65535, "craft_volume_tiled: %d queries per sample exceed the grid", N1);
  CUtensorMap tmA, tmB, tmO;
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)N1, (uint64_t)B};
    uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)N1 * C * 2};
    uint32_t box[3] = {64, 128, 1};
    PFB_TRY(make_tensor_map(&tmA, q1, dtype, 3, dims, str, box));
  }
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {64, 16, 8, 1};
    PFB_TRY(make_tensor_map(&tmB, k2, dtype, 4, dims, str, box));
  }
  TiledOut out{};
  PFB_TRY(tiled_out_maps(pyramid, B, N1, H, W, levels, dtype, &out, &tmO));
  char* ws = reinterpret_cast<char*>(workspace);
  double* partial = reinterpret_cast<double*>(ws);
  float* stats = reinterpret_cast<float*>(ws + align_up(craft_tiled_ctas(B, H, W) * 2 * sizeof(double), 256));
  const size_t smem = (size_t)kCraftChunks * 2 * kTileBytes + acc_tile_bytes(128) + sizeof(CraftBars) + 1024;
  const dim3 grid(n_patches, m_tiles, B);
  const float scale = 1.0f / sqrtf((float)(C / M));
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_VOLUME, s);
  PFB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), s));
  const int nblk = m_tiles * n_patches;
  if (dtype == PFB_F16) {
    PFB_TRY((launch_craft_tiled<__half, 0>(grid, smem, s, tmA, tmB, tmO, out, H, W, N1, M, scale, a, bias, R, flag, clip, partial, stats, levels)));
    PFB_TRY((launch_craft_tiled<__half, 1>(grid, smem, s, tmA, tmB, tmO, out, H, W, N1, M, scale, a, bias, R, flag, clip, partial, stats, levels)));
    volume_stats_kernel<<<B, 32, 0, s>>>(partial, nblk, (size_t)N1 * N1, stats);
    PFB_TRY((launch_craft_tiled<__half, 2>(grid, smem, s, tmA, tmB, tmO, out, H, W, N1, M, scale, a, bias, R, flag, clip, partial, stats, levels)));
  } else {
    PFB_TRY((launch_craft_tiled<__nv_bfloat16, 0>(grid, smem, s, tmA, tmB, tmO, out, H, W, N1, M, scale, a, bias, R, flag, clip, partial, stats, levels)));
    PFB_TRY((launch_craft_tiled<__nv_bfloat16, 1>(grid, smem, s, tmA, tmB, tmO, out, H, W, N1, M, scale, a, bias, R, flag, clip, partial, stats, levels)));
    volume_stats_kernel<<<B, 32, 0, s>>>(partial, nblk, (size_t)N1 * N1, stats);
    PFB_TRY((launch_craft_tiled<__nv_bfloat16, 2>(grid, smem, s, tmA, tmB, tmO, out, H, W, N1, M, scale, a, bias, R, flag, clip, partial, stats, levels)));
  }
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
