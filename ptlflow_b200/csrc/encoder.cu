// Encoder-side kernels (SURVEY.md 8(f) rank 1, first step): the convolutions of BasicEncoder /
// SmallEncoder still run in cuDNN, but everything around them is native and fused --
//   * pfb_preprocess_frames : (x - 0.5) * 2, BGR->RGB, replicate padding, NCHW -> pixel-major, one pass
//                             (raft.py:127-135, base_model.py:206-246)
//   * pfb_instance_norm_act : per-(sample, channel) statistics + normalise + ReLU (+ residual add + ReLU)
//                             (extractor.py:29-31,49-58 -- torch runs this as batch_norm_collect_statistics,
//                             batch_norm_transform_input, relu, add, relu: five passes)
//   * pfb_add_act           : relu(residual + relu(x)) for the batch-norm (folded) context encoder
#include <algorithm>

#include <stdlib.h>

#include "common.cuh"

namespace pfb {

template <typename T>
__global__ void preprocess_frames_kernel(const T* __restrict__ img, T* __restrict__ out, int B, int T_in, int F, int H, int W, int Hp,
                                         int Wp, int pad_top, int pad_left, int OC) {
  // out: [F*B][Hp][Wp][OC], frame-major (all first frames, then all second frames, ...); channels >= 3 are zero
  const size_t total = (size_t)F * B * Hp * Wp;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int x = (int)(idx % Wp);
    size_t t = idx / Wp;
    int y = (int)(t % Hp);
    int n = (int)(t / Hp);
    const int f = n / B, b = n - f * B;
    int sy = y - pad_top, sx = x - pad_left;
    sy = sy < 0 ? 0 : (sy >= H ? H - 1 : sy);
    sx = sx < 0 ? 0 : (sx >= W ? W - 1 : sx);
    const T* src = img + (((size_t)b * T_in + f) * 3) * H * W + (size_t)sy * W + sx;
    T* o = out + idx * OC;
#pragma unroll
    for (int c = 0; c < 3; ++c) {  // output channel c (RGB) <- input channel 2-c (BGR)
      float v = to_f32(src[(size_t)(2 - c) * H * W]);
      o[c] = from_f32<T>((v + (-0.5f)) * 2.0f);
    }
    for (int c = 3; c < OC; ++c) o[c] = from_f32<T>(0.f);
  }
}

// fast path: 4-channel output, no horizontal padding, W % 8 == 0 -> a thread turns 8 pixels (3 x 16-byte plane loads)
// into 8 x 8-byte pixels (4 x 16-byte stores); rows are still replicate-padded vertically
template <typename T>
__global__ void preprocess_frames_vec8_kernel(const T* __restrict__ img, T* __restrict__ out, int B, int T_in, int F, int H, int W, int Hp,
                                              int pad_top) {
  static_assert(sizeof(T) == 2, "16-byte vectors of 2-byte elements");
  const int W8 = W / 8;
  const size_t total = (size_t)F * B * Hp * W8;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int x8 = (int)(idx % W8);
    size_t t = idx / W8;
    const int y = (int)(t % Hp);
    const int n = (int)(t / Hp);
    const int f = n / B, b = n - f * B;
    int sy = y - pad_top;
    sy = sy < 0 ? 0 : (sy >= H ? H - 1 : sy);
    const T* src = img + (((size_t)b * T_in + f) * 3) * H * W + (size_t)sy * W + 8 * x8;
    uint4 pl[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) pl[c] = __ldg(reinterpret_cast<const uint4*>(src + (size_t)(2 - c) * H * W));  // RGB <- BGR planes
    const T* r = reinterpret_cast<const T*>(&pl[0]);
    const T* g = reinterpret_cast<const T*>(&pl[1]);
    const T* bl = reinterpret_cast<const T*>(&pl[2]);
    uint4 o[4];
    T* e = reinterpret_cast<T*>(o);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      e[4 * k + 0] = from_f32<T>((to_f32(r[k]) + (-0.5f)) * 2.0f);
      e[4 * k + 1] = from_f32<T>((to_f32(g[k]) + (-0.5f)) * 2.0f);
      e[4 * k + 2] = from_f32<T>((to_f32(bl[k]) + (-0.5f)) * 2.0f);
      e[4 * k + 3] = from_f32<T>(0.f);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + (idx * 8) * 4);
#pragma unroll
    for (int q = 0; q < 4; ++q) dst[q] = o[q];
  }
}

// ---- instance norm ---------------------------------------------------------------------------------
// stats: [B][C][2] doubles (sum, sum of squares), zeroed by the caller-side memset node.
// thread -> (channel octet, pixel lane): 16-byte loads, consecutive threads on consecutive octets (coalesced);
// per-thread fp32 partials over a few dozen pixels -> shared-memory fp32 atomics per block -> fp64 global atomics.
template <typename T>
__device__ __forceinline__ void load8(const T* p, float (&f)[8]) {
  uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = to_f32(h[i]);
}
template <>
__device__ __forceinline__ void load8<float>(const float* p, float (&f)[8]) {
  float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

template <typename T>
__global__ void __launch_bounds__(256) inorm_stats_kernel(const T* __restrict__ x, double* __restrict__ stats, int HW, int C,
                                                          int pix_per_block) {
  extern __shared__ float acc[];  // [2][C]
  // images in DESCENDING order: blocks are scheduled by increasing index, the producer (a convolution over the whole batch)
  // wrote the last images last, and a 16-frame activation tensor is twice the L2 -- the tail of the batch is still in it
  const int b = gridDim.y - 1 - blockIdx.y;
  const int c8n = C / 8;
  const int lanes = blockDim.x / c8n;
  const int co = threadIdx.x % c8n, pl = threadIdx.x / c8n;
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) acc[i] = 0.f;
  __syncthreads();
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(p0 + pix_per_block, HW);
  float s[8], q[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) s[k] = q[k] = 0.f;
  if (pl < lanes) {
    const T* base = x + (size_t)b * HW * C + 8 * co;
#pragma unroll 4
    for (int p = p0 + pl; p < p1; p += lanes) {
      float v[8];
      load8<T>(base + (size_t)p * C, v);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        s[k] += v[k];
        q[k] = fmaf(v[k], v[k], q[k]);
      }
    }
  }
  // lanes of a warp that own the same channel octet are c8n apart: fold them with shuffles first (when c8n divides
  // 32), so the shared-memory atomics see 32 / c8n times fewer, far less contended, updates
  const bool pow2 = (c8n & (c8n - 1)) == 0 && c8n <= 32 && (blockDim.x % c8n) == 0;
  if (pow2) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      for (int o = c8n; o < 32; o <<= 1) {
        s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
        q[k] += __shfl_xor_sync(0xffffffffu, q[k], o);
      }
    }
  }
  if (pl < lanes && (!pow2 || (threadIdx.x & 31) < c8n)) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      atomicAdd(&acc[8 * co + k], s[k]);
      atomicAdd(&acc[C + 8 * co + k], q[k]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    const int c = i % C, which = i / C;
    atomicAdd(stats + ((size_t)b * C + c) * 2 + which, (double)acc[i]);
  }
}

// y = act(x * scale + shift)  [+ residual -> relu];  scale/shift per (sample, channel) (ss_bstride = C) or per
// channel (ss_bstride = 0).  grid = (pixel slabs, B); a thread owns one channel octet (its 8 scale/shift pairs
// live in registers for the whole slab) and walks pixels with 16-byte loads, four pixels in flight.
template <typename T>
__device__ __forceinline__ void store8(T* p, const float (&f)[8]) {
  uint4 u;
  T* h = reinterpret_cast<T*>(&u);
#pragma unroll
  for (int i = 0; i < 8; ++i) h[i] = from_f32<T>(f[i]);
  *reinterpret_cast<uint4*>(p) = u;
}
template <>
__device__ __forceinline__ void store8<float>(float* p, const float (&f)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}

// scale/shift source: the accumulated instance-norm sums (stats != null: mean / rstd recomputed per thread for its 8
// channels -- two fp64 loads each, cheaper than a separate finalize launch), or a per-channel bias (scale 1).
// Group norm (stats != null and group > 1 or an affine / bias given): the per-channel sums of x are combined over the `group`
// channels of each group, with the producer's per-channel bias folded in analytically (x + bias is what is normalised: a bias
// differs between the channels of a group, so unlike instance norm it is not removed by the mean), then gamma / beta.
template <typename T>
__global__ void __launch_bounds__(256) affine_act_kernel(const T* __restrict__ x, const double* __restrict__ stats,
                                                         const float* __restrict__ bias, const T* __restrict__ residual,
                                                         T* __restrict__ y, int HW, int C, float eps, int relu, int pix_per_block,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta, int group) {
  const int b = blockIdx.y;
  const int c8n = C / 8;
  const int lanes = blockDim.x / c8n;
  const int co = threadIdx.x % c8n, pl = threadIdx.x / c8n;
  __shared__ float2 ss_sm[512];
  const bool gn = stats && (group > 1 || gamma || bias);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {  // one fp64 mean / variance per channel and block, not per thread
    float2 v = make_float2(1.f, bias ? __ldg(bias + c) : 0.f);
    if (gn) {
      const int c0 = c - c % group;
      double s = 0.0, q = 0.0;
      for (int k = c0; k < c0 + group; ++k) {
        const double2 sq = *reinterpret_cast<const double2*>(stats + ((size_t)b * C + k) * 2);
        const double bk = bias ? (double)__ldg(bias + k) : 0.0;
        s += sq.x + bk * HW;
        q += sq.y + 2.0 * bk * sq.x + bk * bk * HW;
      }
      const double n = (double)HW * group;
      const double mean = s / n;
      double var = q / n - mean * mean;
      var = var < 0 ? 0 : var;
      const double rstd = (double)rsqrtf((float)var + eps);
      const double g = gamma ? (double)__ldg(gamma + c) : 1.0, be = beta ? (double)__ldg(beta + c) : 0.0;
      const double bc = bias ? (double)__ldg(bias + c) : 0.0;
      v = make_float2((float)(rstd * g), (float)((bc - mean) * rstd * g + be));
    } else if (stats) {
      const double2 sq = *reinterpret_cast<const double2*>(stats + ((size_t)b * C + c) * 2);
      const double mean = sq.x / HW;
      double var = sq.y / HW - mean * mean;
      var = var < 0 ? 0 : var;
      const float rstd = rsqrtf((float)var + eps);
      v = make_float2(rstd, (float)(-mean) * rstd);
    }
    ss_sm[c] = v;
  }
  __syncthreads();
  if (pl >= lanes) return;
  float sc[8], sh[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sc[k] = ss_sm[8 * co + k].x;
    sh[k] = ss_sm[8 * co + k].y;
  }
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = min(p0 + pix_per_block, HW);
  const size_t base = (size_t)b * HW * C + 8 * co;
#pragma unroll 4
  for (int p = p0 + pl; p < p1; p += lanes) {
    const size_t off = base + (size_t)p * C;
    float v[8], r[8];
    load8<T>(x + off, v);
    if (residual) load8<T>(residual + off, r);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float o = fmaf(v[k], sc[k], sh[k]);
      if (relu) o = fmaxf(o, 0.f);
      if (residual) o = fmaxf(r[k] + o, 0.f);
      v[k] = o;
    }
    store8<T>(y + off, v);
  }
}

// ---- instance norm, one kernel, one HBM read ------------------------------------------------------------------
// Statistics and normalisation of the SAME image back to back, so the second read of the image comes from L2: the grid is
// `ipw` images x `G` CTAs (one wave of the machine, all co-resident); the G CTAs of an image reduce their pixel slices,
// meet at a per-image counter in global memory, then normalise their slices.  `ipw` is chosen so that the images of a wave
// (input + output) fit the L2.  The two-kernel form reads every activation tensor twice from HBM (16 frames x 220 x 512 x
// 64 channels = 230 MB per layer-1 tensor, twice the 126 MB L2): 0.48 ms of statistics passes per step (bench r02c).
template <typename T>
__global__ void __launch_bounds__(256) inorm_fused_kernel(const T* __restrict__ x, const T* __restrict__ residual, T* __restrict__ y,
                                                          double* __restrict__ stats, unsigned* __restrict__ counters, int B, int HW, int C,
                                                          float eps, int relu, int G, int ipw) {
  extern __shared__ float acc[];  // [2][C] partial sums, then [2][C] scale / shift
  const int iw = blockIdx.x / G, g = blockIdx.x - iw * G;
  const int c8n = C / 8;
  const int lanes = blockDim.x / c8n;
  const int co = threadIdx.x % c8n, pl = threadIdx.x / c8n;
  const int slice = (HW + G - 1) / G;
  const int p0 = g * slice, p1 = min(p0 + slice, HW);
  const bool pow2 = (c8n & (c8n - 1)) == 0 && c8n <= 32 && (blockDim.x % c8n) == 0;
  for (int b = iw; b < B; b += ipw) {
    // ---- phase 1: sums of this CTA's slice ----
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) acc[i] = 0.f;
    __syncthreads();
    const size_t base = (size_t)b * HW * C + 8 * co;
    float s[8], q[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = q[k] = 0.f;
    if (pl < lanes) {
#pragma unroll 4
      for (int p = p0 + pl; p < p1; p += lanes) {
        float v[8];
        load8<T>(x + base + (size_t)p * C, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          s[k] += v[k];
          q[k] = fmaf(v[k], v[k], q[k]);
        }
      }
    }
    if (pow2) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        for (int o = c8n; o < 32; o <<= 1) {
          s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
          q[k] += __shfl_xor_sync(0xffffffffu, q[k], o);
        }
      }
    }
    if (pl < lanes && (!pow2 || (threadIdx.x & 31) < c8n)) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        atomicAdd(&acc[8 * co + k], s[k]);
        atomicAdd(&acc[C + 8 * co + k], q[k]);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
      const int c = i % C, which = i / C;
      atomicAdd(stats + ((size_t)b * C + c) * 2 + which, (double)acc[i]);
    }
    __threadfence();
    __syncthreads();
    // ---- meet the other CTAs of this image ----
    if (threadIdx.x == 0) {
      atomicAdd(counters + b, 1u);
      const unsigned long long t0 = clock64();
      while (*reinterpret_cast<volatile unsigned*>(counters + b) < (unsigned)G) {
        __nanosleep(64);
        if (clock64() - t0 > 4000000000ull) __trap();  // ~2 s: a scheduling assumption failed -- an error, never a hang
      }
      __threadfence();
    }
    __syncthreads();
    // ---- phase 2: scale / shift of the image, then this CTA's slice again (L2) ----
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const double sum = __ldcg(stats + ((size_t)b * C + c) * 2), sq = __ldcg(stats + ((size_t)b * C + c) * 2 + 1);
      const double mean = sum / HW;
      double var = sq / HW - mean * mean;
      var = var < 0 ? 0 : var;
      const float rstd = rsqrtf((float)var + eps);
      acc[c] = rstd;
      acc[C + c] = (float)(-mean) * rstd;
    }
    __syncthreads();
    if (pl < lanes) {
      float sc[8], sh[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        sc[k] = acc[8 * co + k];
        sh[k] = acc[C + 8 * co + k];
      }
#pragma unroll 4
      for (int p = p0 + pl; p < p1; p += lanes) {
        const size_t off = base + (size_t)p * C;
        float v[8], r[8];
        load8<T>(x + off, v);
        if (residual) load8<T>(residual + off, r);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          float o = fmaf(v[k], sc[k], sh[k]);
          if (relu) o = fmaxf(o, 0.f);
          if (residual) o = fmaxf(r[k] + o, 0.f);
          v[k] = o;
        }
        store8<T>(y + off, v);
      }
    }
    __syncthreads();
  }
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_preprocess_frames_ex(const void* images, void* out, int B, int T, int F, int H, int W, int Hp, int Wp, int pad_top,
                                                int pad_left, int out_channels, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(images && out, "preprocess_frames: null pointer");
  PFB_CHECK_ARG(out_channels >= 3 && out_channels <= 16, "preprocess_frames: out_channels=%d (3..16)", out_channels);
  PFB_CHECK_ARG(F >= 1 && T >= F, "preprocess_frames: %d of %d frames", F, T);
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0 && Hp >= H && Wp >= W && pad_top >= 0 && pad_left >= 0 &&
                    pad_top + H <= Hp && pad_left + W <= Wp,
                "preprocess_frames: bad geometry %dx%d -> %dx%d (+%d,+%d)", H, W, Hp, Wp, pad_top, pad_left);
  cudaStream_t s = as_stream(stream);
  size_t total = (size_t)F * B * Hp * Wp;
  unsigned blocks = (unsigned)std::min<size_t>(ceil_div_sz(total, 256), (size_t)sm_count() * 16);
  ProfScope prof(KC_MISC, s);
  if (dtype != PFB_F32 && out_channels == 4 && pad_left == 0 && Wp == W && W % 8 == 0 &&
      ((reinterpret_cast<uintptr_t>(images) | reinterpret_cast<uintptr_t>(out)) & 15) == 0 && ((size_t)H * W) % 8 == 0) {
    blocks = (unsigned)std::min<size_t>(ceil_div_sz(total / 8, 256), (size_t)sm_count() * 16);
    if (dtype == PFB_F16)
      preprocess_frames_vec8_kernel<__half><<<blocks, 256, 0, s>>>((const __half*)images, (__half*)out, B, T, F, H, W, Hp, pad_top);
    else
      preprocess_frames_vec8_kernel<__nv_bfloat16><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)images, (__nv_bfloat16*)out, B, T, F, H, W,
                                                                          Hp, pad_top);
    PFB_LAUNCH_CHECK();
    return PFB_OK;
  }
  PFB_DISPATCH_DTYPE(dtype, T_, {
    preprocess_frames_kernel<T_><<<blocks, 256, 0, s>>>((const T_*)images, (T_*)out, B, T, F, H, W, Hp, Wp, pad_top, pad_left, out_channels);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_preprocess_frames(const void* images, void* out, int B, int H, int W, int Hp, int Wp, int pad_top,
                                             int pad_left, int out_channels, pfb_dtype dtype, pfb_stream stream) {
  return pfb_preprocess_frames_ex(images, out, B, 2, 2, H, W, Hp, Wp, pad_top, pad_left, out_channels, dtype, stream);
}

extern "C" PFB_API size_t pfb_instance_norm_workspace_bytes(int B, int C) {
  return (size_t)B * C * (2 * sizeof(double) + sizeof(float2));
}

template <typename T>
static int launch_affine(const void* x, const double* stats, const float* bias, const void* residual, void* y, int B, int HW, int C,
                         float eps, int relu, cudaStream_t s, const float* gamma = nullptr, const float* beta = nullptr, int group = 1) {
  const int ppb = HW >= 8192 ? 512 : (HW >= 1024 ? 128 : 32);
  dim3 grid(ceil_div(HW, ppb), B);
  affine_act_kernel<T><<<grid, 256, 0, s>>>((const T*)x, stats, bias, (const T*)residual, (T*)y, HW, C, eps, relu, ppb, gamma, beta, group);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

// per-(image, channel) sums of x into the zeroed workspace (instance norm and group norm share them)
static int launch_stats(const void* x, double* stats, int B, int HW, int C, pfb_dtype dtype, cudaStream_t s) {
  // plenty of blocks, few global atomics (fewer, fatter blocks were measured slower: r01 launch list v19)
  const int threads = 256;
  static const int env_ppb = getenv("PFB_STATS_PPB") ? atoi(getenv("PFB_STATS_PPB")) : 0;  // tuning knob
  const int ppb = env_ppb > 0 && HW >= 8192 ? env_ppb : (HW >= 65536 ? 1536 : (HW >= 8192 ? 768 : (HW >= 1024 ? 256 : 64)));
  dim3 grid(ceil_div(HW, ppb), B);
  ProfScope prof(KC_ENC_STATS, s);
  PFB_DISPATCH_DTYPE(dtype, T, { inorm_stats_kernel<T><<<grid, threads, 2 * C * sizeof(float), s>>>((const T*)x, stats, HW, C, ppb); });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_instance_norm_act(const void* x, void* y, const void* residual, void* workspace, int B, int H, int W,
                                             int C, float eps, int relu, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && y && workspace, "instance_norm_act: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && C <= 512,
                "instance_norm_act: bad shape (C=%d must be a multiple of 8, <= 512)", C);
  cudaStream_t s = as_stream(stream);
  const int HW = H * W;
  double* stats = reinterpret_cast<double*>(workspace);
  // sums, and (fused kernel) one arrival counter per image right behind them: the scale / shift area of the workspace
  PFB_CUDA(cudaMemsetAsync(stats, 0, (size_t)B * C * 2 * sizeof(double) + (size_t)B * sizeof(unsigned), s));
  PFB_CHECK_ARG(B <= 65535, "instance_norm_act: batch too large");
  {
    // opt-in: measured 3.15 ms per step against 1.19 + 0.49 ms for the two-kernel form (bench r02e) -- one co-resident wave of
    // 256-thread CTAs keeps too few loads in flight to stream from HBM, which costs more than the second read saves
    static const int env_fused = getenv("PFB_INORM_FUSED") ? atoi(getenv("PFB_INORM_FUSED")) : 0;
    const size_t image_bytes = (size_t)HW * C * dtype_size(dtype);
    if (env_fused && dtype != PFB_F32 && C <= 256 && (256 % (C / 8) == 0 || C / 8 <= 32) && HW >= 1024) {
      // images per wave: input + output (+ residual) of a wave within ~half of the 126 MB L2; at least 2 CTAs per image
      const size_t per_image = image_bytes * (residual ? 3 : 2);
      int ipw = (int)std::max<size_t>(1, std::min<size_t>((size_t)B, (size_t)(60u << 20) / std::max<size_t>(per_image, 1)));
      const int sms = sm_count();
      if (ipw > sms / 2) ipw = sms / 2;
      const int G = std::max(1, sms / ipw);
      unsigned* counters = reinterpret_cast<unsigned*>(stats + (size_t)B * C * 2);
      ProfScope prof(KC_ENC_AFFINE, s);
      PFB_DISPATCH_DTYPE(dtype, T, {
        inorm_fused_kernel<T><<<ipw * G, 256, 2 * C * sizeof(float), s>>>((const T*)x, (const T*)residual, (T*)y, stats, counters, B, HW, C, eps,
                                                                        relu, G, ipw);
      });
      PFB_LAUNCH_CHECK();
      return PFB_OK;
    }
  }
  int rc = launch_stats(x, stats, B, HW, C, dtype, s);
  if (rc != PFB_OK) return rc;
  ProfScope prof(KC_ENC_AFFINE, s);
  PFB_DISPATCH_DTYPE(dtype, T, { return launch_affine<T>(x, stats, nullptr, residual, y, B, HW, C, eps, relu, s); });
  return PFB_OK;
}

// Second half of pfb_instance_norm_act for a producer that already accumulated the sums (pfb_first_conv7x7s2):
// workspace = [B*C*2 doubles (sum, sum of squares)] [B*C float2 scale/shift]
extern "C" PFB_API int pfb_instance_norm_apply(const void* x, void* y, const void* residual, void* workspace, int B, int H, int W,
                                               int C, float eps, int relu, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && y && workspace, "instance_norm_apply: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && C <= 512 && B <= 65535,
                "instance_norm_apply: bad shape (C=%d must be a multiple of 8, <= 512)", C);
  cudaStream_t s = as_stream(stream);
  const int HW = H * W;
  double* stats = reinterpret_cast<double*>(workspace);
  ProfScope prof(KC_ENC_AFFINE, s);
  PFB_DISPATCH_DTYPE(dtype, T, { return launch_affine<T>(x, stats, nullptr, residual, y, B, HW, C, eps, relu, s); });
  return PFB_OK;
}

static int check_group_norm(const void* x, const void* y, const void* workspace, int B, int H, int W, int C, int group_size,
                            pfb_dtype dtype, const char* what) {
  PFB_CHECK_ARG(x && y && workspace, "%s: null pointer", what);
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && C <= 512 && B <= 65535,
                "%s: bad shape (C=%d must be a multiple of 8, <= 512)", what, C);
  PFB_CHECK_ARG(group_size >= 1 && C % group_size == 0, "%s: group_size=%d must divide C=%d", what, group_size, C);
  return PFB_OK;
}

// Group norm: statistics per (image, group of group_size channels) of x + bias, then gamma / beta, then act / residual join.
extern "C" PFB_API int pfb_group_norm_act(const void* x, void* y, const void* residual, void* workspace, const float* bias,
                                          const float* gamma, const float* beta, int B, int H, int W, int C, int group_size, float eps,
                                          int relu, pfb_dtype dtype, pfb_stream stream) {
  int rc = check_group_norm(x, y, workspace, B, H, W, C, group_size, dtype, "group_norm_act");
  if (rc != PFB_OK) return rc;
  cudaStream_t s = as_stream(stream);
  double* stats = reinterpret_cast<double*>(workspace);
  PFB_CUDA(cudaMemsetAsync(stats, 0, (size_t)B * C * 2 * sizeof(double), s));
  rc = launch_stats(x, stats, B, H * W, C, dtype, s);
  if (rc != PFB_OK) return rc;
  ProfScope prof(KC_ENC_AFFINE, s);
  PFB_DISPATCH_DTYPE(dtype, T, { return launch_affine<T>(x, stats, bias, residual, y, B, H * W, C, eps, relu, s, gamma, beta, group_size); });
  return PFB_OK;
}

extern "C" PFB_API int pfb_group_norm_apply(const void* x, void* y, const void* residual, void* workspace, const float* bias,
                                            const float* gamma, const float* beta, int B, int H, int W, int C, int group_size, float eps,
                                            int relu, pfb_dtype dtype, pfb_stream stream) {
  int rc = check_group_norm(x, y, workspace, B, H, W, C, group_size, dtype, "group_norm_apply");
  if (rc != PFB_OK) return rc;
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_ENC_AFFINE, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    return launch_affine<T>(x, reinterpret_cast<const double*>(workspace), bias, residual, y, B, H * W, C, eps, relu, s, gamma, beta,
                            group_size);
  });
  return PFB_OK;
}

// y = act(x + bias[c]) [+ residual -> relu]; bias fp32 [C] or NULL; workspace >= C * 8 bytes
extern "C" PFB_API int pfb_bias_act(const void* x, const float* bias, const void* residual, void* y, void* workspace, int B, int H,
                                    int W, int C, int relu, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && y && workspace, "bias_act: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && C <= 512, "bias_act: bad shape (C=%d must be a multiple of 8, <= 512)", C);
  PFB_CHECK_ARG(B <= 65535, "bias_act: batch too large");
  cudaStream_t s = as_stream(stream);
  (void)workspace;
  ProfScope prof(KC_ENC_AFFINE, s);
  PFB_DISPATCH_DTYPE(dtype, T, { return launch_affine<T>(x, nullptr, bias, residual, y, B, H * W, C, 0.f, relu, s); });
  return PFB_OK;
}
