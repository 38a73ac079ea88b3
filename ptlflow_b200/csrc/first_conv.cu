// First encoder convolution (7x7, stride 2, 3 -> 64 channels; ptlflow/models/raft/extractor.py:136,171-178) on the
// Hopper tensor cores (wgmma) WITHOUT an im2col buffer.
//
//   out[n, y, x, co] = sum_{ky, kx, c} X[n, 2y + ky - 3, 2x + kx - 3, c] * W[co, c, ky, kx]        (zero padding 3)
//
// The frames arrive pixel-major with 4 channels (RGB + a zero channel: 8-byte pixels).  For one input row r the
// 8-pixel window of output pixel x, input pixels 2x-4 .. 2x+3, is 64 contiguous bytes that start 16 bytes after
// the window of pixel x-1.  That is exactly the geometry of a NON-swizzled K-major wgmma operand whose "core
// matrices" (8 rows x 16 bytes, rows 16 bytes apart) overlap: leading-dimension (K) byte offset 16, stride (N)
// byte offset 128.  So the B operand of wgmma is the raw input row in shared memory, read through an
// overlapping-window descriptor: N = 128 output pixels, K = 32 (8 pixels x 4 channels) per input row.
// The weights are the A operand: M = 128 = 64 output channels x 2 output rows (rows y and y+1 of a pair see input
// row r through filter rows ky and ky-2), packed per input-row offset j = r - (2y - 3), j = 0..8, as canonical
// non-swizzled K-major tiles [16 row groups][4 K groups][8 rows][16 B] by the host (models/raft/extractor.py); two
// warpgroups take the two row phases (M = 64 each).
// The accumulator is TRANSPOSED (row = (row phase, channel), column = pixel), which makes the per-channel
// instance-norm statistics a per-thread reduction: they are accumulated from the fp32 accumulators in the
// epilogue, so the separate statistics pass over the 230 MB activation tensor disappears, and for the
// batch-norm (folded) encoder bias + ReLU are applied here and nothing else touches the tensor.
//
// 18 K steps (128 x 128 x 16) per work item (= 2 output rows x 128 pixels), 19 KB of input rows per item.  The item
// width is what lets the fp32 accumulator tile (64 KB) sit in shared memory next to the weights and two input slots.
#include <stdlib.h>

#include <type_traits>

#include "umma.cuh"

namespace pfb {
using namespace sm90;

constexpr int kFcPix = 128;        // output pixels per work item (the N of the MMA)
constexpr int kFcRowBytes = 2176;  // (2 * 128 + 8) pixels * 8 B = 2112, + zero tail, 128-byte multiple
constexpr int kFcRows = 9;
constexpr int kFcSlotBytes = kFcRows * kFcRowBytes;
constexpr int kFcABytes = 9 * 8192;
constexpr int kFcSlots = 2;

struct __align__(8) FcBars {
  uint64_t full[kFcSlots];
  uint64_t empty[kFcSlots];
  uint64_t acc_full;
  uint64_t acc_empty;
  uint64_t a_full;
};

struct FcArgs {
  const void* x;      // [N][H][W][4]
  const void* wpack;  // [9][8192 B]
  void* out;          // [N][Ho][Wo][64]
  const float* bias;  // [64] or null
  double* stats;      // [N][64][2] (sum, sum of squares of the fp32 accumulator + bias) or null
  int N, H, W, Ho, Wo;
  int pairs, nseg, n_items, per_cta;
  int relu, ab_fmt;
};

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Epilogue store of one 32-pixel x 32-channel chunk held transposed (lane = channel, v[e] = pixel e): 2-byte global
// stores (32 per lane, one 64-byte segment per warp instruction) made the first version store-issue bound (ncu launch
// list r01 v18: 118 us per launch against ~25 us of MMA time).  Staged through 2 KB of warp-private shared memory
// instead and written as 16-byte vectors: 4 stores per lane.
template <typename T>
__device__ __forceinline__ void store_chunk_transposed(uint8_t* stage, const float (&v)[32], T* gbase, size_t pix_stride, int npx_valid,
                                                       int lane) {
  T* st = reinterpret_cast<T*>(stage);
#pragma unroll
  for (int e = 0; e < 32; ++e) st[e * 32 + lane] = from_f32<T>(v[e]);
  __syncwarp();
  const int part = lane & 3;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int px = (lane >> 2) + 8 * k;
    if (px < npx_valid) *reinterpret_cast<uint4*>(gbase + (size_t)px * pix_stride + part * 8) = *reinterpret_cast<const uint4*>(stage + px * 64 + part * 16);
  }
  __syncwarp();
}

// 17 warps: 0-7 epilogue, 8-15 the two MMA warpgroups (row phase 0 / 1), 16 producer
constexpr int kFcThreads = 17 * 32;
template <typename T>
__global__ void __launch_bounds__(kFcThreads, 1) first_conv_umma_kernel(const FcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemX = smem + kFcABytes;
  float* sacc = reinterpret_cast<float*>(smemX + kFcSlots * kFcSlotBytes);  // fp32 accumulator tile, kFcPix columns
  uint8_t* smemStage = reinterpret_cast<uint8_t*>(sacc) + acc_tile_bytes(kFcPix);  // 8 epilogue warps x 2 KB
  FcBars* bars = reinterpret_cast<FcBars*>(smemStage + 8 * 2048);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kFcSlots; ++s) {
      mbar_init(&bars->full[s], 1);
      mbar_init(&bars->empty[s], 8);  // one arrival per MMA warp
    }
    mbar_init(&bars->acc_full, 8);
    mbar_init(&bars->acc_empty, 8);  // one arrival per epilogue warp
    mbar_init(&bars->a_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  const int w0 = blockIdx.x * a.per_cta;
  const int w1 = min(a.n_items, w0 + a.per_cta);
  auto decode = [&](int w, int& n, int& y, int& x0) {
    const int per_img = a.pairs * a.nseg;
    n = w / per_img;
    const int r = w - n * per_img;
    const int q = r / a.nseg;
    y = 2 * q;
    x0 = (r - q * a.nseg) * kFcPix;
  };

  if (warp == 16) {
    // ================= producer: weights once, then 9 input rows per item (1-D bulk copies) =================
    if (lane == 0) {
      mbar_arrive_expect_tx(&bars->a_full, kFcABytes);
      for (int j = 0; j < 9; ++j) bulk_g2s(smemA + j * 8192, reinterpret_cast<const uint8_t*>(a.wpack) + j * 8192, 8192, &bars->a_full);
    }
    int i = 0;
    for (int w = w0; w < w1; ++w, ++i) {
      int n, y, x0;
      decode(w, n, y, x0);
      const int slot = i % kFcSlots;
      mbar_wait(&bars->empty[slot], ((i / kFcSlots) & 1) ^ 1);
      uint8_t* base = smemX + slot * kFcSlotBytes;
      // pixels [plo, phi) of the row are copied to byte (plo - (2*x0 - 4)) * 8 of the row buffer; what the windows of
      // valid outputs can touch outside the image is zeroed (generic-proxy stores, fenced before the hand-off)
      const int pstart = 2 * x0 - 4;
      const int plo = pstart < 0 ? 0 : pstart;
      int phi = 2 * x0 + 2 * kFcPix + 2;
      if (phi > a.W) phi = a.W;
      const uint32_t bytes = (uint32_t)(phi - plo) * 8u;
      const uint32_t doff = (uint32_t)(plo - pstart) * 8u;
      const int r0 = 2 * y - 3;
      if (lane < kFcRows) {
        uint8_t* row = base + lane * kFcRowBytes;
        if (doff) {
          reinterpret_cast<uint4*>(row)[0] = make_uint4(0u, 0u, 0u, 0u);
          reinterpret_cast<uint4*>(row)[1] = make_uint4(0u, 0u, 0u, 0u);
        }
        reinterpret_cast<uint4*>(row + doff + bytes)[0] = make_uint4(0u, 0u, 0u, 0u);
        reinterpret_cast<uint4*>(row + doff + bytes)[1] = make_uint4(0u, 0u, 0u, 0u);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        int nvalid = 0;
        for (int j = 0; j < kFcRows; ++j) nvalid += (r0 + j >= 0 && r0 + j < a.H);
        mbar_arrive_expect_tx(&bars->full[slot], bytes * nvalid);
        for (int j = 0; j < kFcRows; ++j) {
          const int r = r0 + j;
          if (r < 0 || r >= a.H) continue;
          const uint8_t* src = reinterpret_cast<const uint8_t*>(a.x) + (((size_t)n * a.H + r) * a.W + plo) * 8;
          bulk_g2s(base + j * kFcRowBytes + doff, src, bytes, &bars->full[slot]);
        }
      }
      __syncwarp();
    }
  } else if (warp >= 8) {
    // ================= MMA warpgroups: rows 0-63 (output row y) and 64-127 (row y + 1) =================
    // non-swizzled K-major descriptors: LBO = byte distance between core matrices along K, SBO = along M / N
    // (tests/test_gpu_ops.py::test_first_conv7x7s2_vs_torch checks the reading)
    const int wg = (threadIdx.x >> 7) - 2, tid = threadIdx.x & 127;
    const uint32_t a_hi = gdesc_hi(512, 0), b_hi = gdesc_hi(128, 0);
    const uint32_t a_lo0 = gdesc_lo(smem_u32(smemA) + wg * 4096, 128);
    mbar_wait(&bars->a_full, 0);
    float d[kFcPix / 2];
    int i = 0;
    for (int w = w0; w < w1; ++w, ++i) {
      int n, y, x0;
      decode(w, n, y, x0);
      const int slot = i % kFcSlots;
      mbar_wait(&bars->full[slot], (i / kFcSlots) & 1);
      const uint32_t b_lo0 = gdesc_lo(smem_u32(smemX + slot * kFcSlotBytes), 16);
      const int r0 = 2 * y - 3;
      uint32_t acc = 0;
      wgmma_fence();
      for (int j = 0; j < kFcRows; ++j) {
        if (r0 + j < 0 || r0 + j >= a.H) continue;  // rows outside the image contribute zero
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          wgmma<kFcPix, std::is_same<T, __nv_bfloat16>::value>(d, gdesc(a_lo0 + ((j * 8192 + s * 256) >> 4), a_hi),
                                                               gdesc(b_lo0 + ((j * kFcRowBytes + s * 32) >> 4), b_hi), acc);
          acc = 1;
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(d);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->empty[slot]);
      mbar_wait(&bars->acc_empty, (i & 1) ^ 1);
      acc_store<kFcPix>(sacc, d, wg * 64, tid);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->acc_full);
    }
  } else {
    // ================= epilogue: row = (row phase p, channel co), columns = pixels =================
    // 8 epilogue warps: two column groups x four row quarters.  Each warp owns two 32-pixel chunks of an item; both are read
    // before the accumulator tile is handed back to the MMA warpgroups.
    const int quarter = warp & 3, group = warp >> 2;
    const int m = quarter * 32 + lane;
    const int p = m >> 6, co = m & 63;
    const float bias = a.bias ? a.bias[co] : 0.f;
    uint8_t* stage = smemStage + warp * 2048;
    float ssum = 0.f, ssq = 0.f;
    int n_cur = -1;
    auto flush = [&]() {
      if (a.stats && n_cur >= 0) {
        atomicAdd(&a.stats[((size_t)n_cur * 64 + co) * 2 + 0], (double)ssum);
        atomicAdd(&a.stats[((size_t)n_cur * 64 + co) * 2 + 1], (double)ssq);
      }
      ssum = 0.f;
      ssq = 0.f;
    };
    int i = 0;
    for (int w = w0; w < w1; ++w, ++i) {
      int n, y, x0;
      decode(w, n, y, x0);
      if (n != n_cur) {
        flush();
        n_cur = n;
      }
      const bool row_ok = (y + p) < a.Ho;
      // this warp's 32 channels of the output row: channel offset (quarter & 1) * 32
      T* orow32 = reinterpret_cast<T*>(a.out) + (((size_t)n * a.Ho + (row_ok ? y + p : 0)) * a.Wo) * 64 + (quarter & 1) * 32;
      mbar_wait(&bars->acc_full, i & 1);
      uint32_t r[2][32];
      acc_ld32(sacc, m, group * 32, r[0]);
      acc_ld32(sacc, m, group * 32 + 64, r[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->acc_empty);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int xb = x0 + group * 32 + 64 * k;
        if (!row_ok || xb >= a.Wo) continue;  // warp-uniform
        const int nv = a.Wo - xb;
        float v[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) {
          v[e] = __uint_as_float(r[k][e]) + bias;
          if (e < nv) {
            ssum += v[e];
            ssq = fmaf(v[e], v[e], ssq);
          }
          if (a.relu) v[e] = fmaxf(v[e], 0.f);
        }
        store_chunk_transposed<T>(stage, v, orow32 + (size_t)xb * 64, 64, nv, lane);
      }
    }
    flush();
  }
}


// ------------------------------------------------------------------------------------------------------------
// convf1 of the motion encoder: nn.Conv2d(2, 128, 7, padding=3) on the current flow (update.py:84,96), every
// iteration.  Same overlapping-window trick with stride 1: the fp32 flow is split into hi + lo halves of the storage
// type (fx_hi, fy_hi, fx_lo, fy_lo, 0, 0, 0, 0 = one 16-byte pixel, so no precision is lost against the fp32 SIMT
// kernel it replaces), output pixel x reads pixels x-4 .. x+3 = 128 contiguous bytes, 16 bytes after pixel x-1's.
// M = 128 output channels (two warpgroups of 64), N = 128 pixel columns (one image row segment), K = 64 per filter row.
// Loader warps build the split rows in shared memory (generic stores + fence.proxy.async): no global staging buffer.
struct FlowConvArgs {
  const float* flow;  // [B][H][W][2]
  const void* wpack;  // [7][16384 B]
  const float* bias;  // [128]
  void* out;          // [B][H][W][out_stride], channels out_offset .. out_offset + 127
  int B, H, W, out_stride, out_offset;
  int nseg, n_items, per_cta, ab_fmt;
};
constexpr int kFlRows = 7;
constexpr int kFlSlotBytes = kFlRows * kFcRowBytes;  // (128 + 8) pixels x 16 B per row
constexpr int kFlABytes = 7 * 16384;
constexpr int kFlLoaders = 128;

struct __align__(8) FlBars {
  uint64_t full[2];
  uint64_t empty[2];
  uint64_t acc_full;
  uint64_t acc_empty;
  uint64_t a_full;
};

template <typename T>
__device__ __forceinline__ uint4 split_flow(float fx, float fy) {
  const T hx = from_f32<T>(fx), hy = from_f32<T>(fy);
  const T lx = from_f32<T>(fx - to_f32(hx)), ly = from_f32<T>(fy - to_f32(hy));
  uint4 u;
  u.x = (uint32_t)(*reinterpret_cast<const uint16_t*>(&hx)) | ((uint32_t)(*reinterpret_cast<const uint16_t*>(&hy)) << 16);
  u.y = (uint32_t)(*reinterpret_cast<const uint16_t*>(&lx)) | ((uint32_t)(*reinterpret_cast<const uint16_t*>(&ly)) << 16);
  u.z = 0u;
  u.w = 0u;
  return u;
}

// 20 warps: 0-7 epilogue, 8-15 the two MMA warpgroups, 16-19 loaders
constexpr int kFlThreads = 20 * 32;
template <typename T>
__global__ void __launch_bounds__(kFlThreads, 1) flow_conv7x7_umma_kernel(const FlowConvArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemX = smem + kFlABytes;
  float* sacc = reinterpret_cast<float*>(smemX + 2 * kFlSlotBytes);  // fp32 accumulator tile, kFcPix columns
  uint8_t* smemStage = reinterpret_cast<uint8_t*>(sacc) + acc_tile_bytes(kFcPix);  // 8 epilogue warps x 2 KB
  FlBars* bars = reinterpret_cast<FlBars*>(smemStage + 8 * 2048);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bars->full[s], kFlLoaders);
      mbar_init(&bars->empty[s], 8);  // one arrival per MMA warp
    }
    mbar_init(&bars->acc_full, 8);
    mbar_init(&bars->acc_empty, 8);  // one arrival per epilogue warp
    mbar_init(&bars->a_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  // the weights do not depend on the previous kernel: request them before the PDL wait
  if (warp == 16 && lane == 0) {
    mbar_arrive_expect_tx(&bars->a_full, kFlABytes);
    for (int j = 0; j < 7; ++j) bulk_g2s(smemA + j * 16384, reinterpret_cast<const uint8_t*>(a.wpack) + j * 16384, 16384, &bars->a_full);
  }
  pdl_wait();
  pdl_trigger();

  const int w0 = blockIdx.x * a.per_cta;
  const int w1 = min(a.n_items, w0 + a.per_cta);
  auto decode = [&](int w, int& n, int& y, int& x0) {
    const int row = w / a.nseg;
    x0 = (w - row * a.nseg) * kFcPix;
    n = row / a.H;
    y = row - n * a.H;
  };

  if (warp >= 16) {
    // ================= loaders: fp32 flow rows -> split 16-byte pixels with zero halo =================
    const int t = threadIdx.x - 512;  // 0..127
    int i = 0;
    for (int w = w0; w < w1; ++w, ++i) {
      int n, y, x0;
      decode(w, n, y, x0);
      const int slot = i & 1;
      mbar_wait(&bars->empty[slot], ((i >> 1) & 1) ^ 1);
      uint8_t* base = smemX + slot * kFlSlotBytes;
      // buffer pixel i <-> image pixel x0 - 4 + i, i in [0, kFcPix + 8)
      for (int e = t; e < kFlRows * (kFcPix + 8); e += kFlLoaders) {
        const int j = e / (kFcPix + 8), bi = e - j * (kFcPix + 8);
        const int r = y + j - 3, px = x0 - 4 + bi;
        uint4 u = make_uint4(0u, 0u, 0u, 0u);
        if (r >= 0 && r < a.H && px >= 0 && px < a.W) {
          const float2 f = __ldg(reinterpret_cast<const float2*>(a.flow) + ((size_t)n * a.H + r) * a.W + px);
          u = split_flow<T>(f.x, f.y);
        }
        *reinterpret_cast<uint4*>(base + j * kFcRowBytes + bi * 16) = u;
      }
      fence_proxy_async();
      mbar_arrive(&bars->full[slot]);
    }
  } else if (warp >= 8) {
    // ================= MMA warpgroups: output channels 0-63 and 64-127 =================
    const int wg = (threadIdx.x >> 7) - 2, tid = threadIdx.x & 127;
    const uint32_t a_hi = gdesc_hi(1024, 0), b_hi = gdesc_hi(128, 0);
    const uint32_t a_lo0 = gdesc_lo(smem_u32(smemA) + wg * 8192, 128);
    mbar_wait(&bars->a_full, 0);
    float d[kFcPix / 2];
    int i = 0;
    for (int w = w0; w < w1; ++w, ++i) {
      int n, y, x0;
      decode(w, n, y, x0);
      const int slot = i & 1;
      mbar_wait(&bars->full[slot], (i >> 1) & 1);
      const uint32_t b_lo0 = gdesc_lo(smem_u32(smemX + slot * kFlSlotBytes), 16);
      uint32_t acc = 0;
      wgmma_fence();
      for (int j = 0; j < kFlRows; ++j) {
        if (y + j - 3 < 0 || y + j - 3 >= a.H) continue;  // rows outside the image are zero
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          wgmma<kFcPix, std::is_same<T, __nv_bfloat16>::value>(d, gdesc(a_lo0 + ((j * 16384 + s * 256) >> 4), a_hi),
                                                               gdesc(b_lo0 + ((j * kFcRowBytes + s * 32) >> 4), b_hi), acc);
          acc = 1;
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(d);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->empty[slot]);
      mbar_wait(&bars->acc_empty, (i & 1) ^ 1);
      acc_store<kFcPix>(sacc, d, wg * 64, tid);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->acc_full);
    }
  } else {
    // ================= epilogue: row = output channel, columns = pixels =================
    const int quarter = warp & 3, group = warp >> 2;
    const int co = quarter * 32 + lane;
    const float bias = a.bias ? a.bias[co] : 0.f;
    uint8_t* stage = smemStage + warp * 2048;
    int i = 0;
    for (int w = w0; w < w1; ++w, ++i) {
      int n, y, x0;
      decode(w, n, y, x0);
      T* orow32 = reinterpret_cast<T*>(a.out) + (((size_t)n * a.H + y) * a.W) * a.out_stride + a.out_offset + quarter * 32;
      mbar_wait(&bars->acc_full, i & 1);
      for (int c = group * 32; c < kFcPix && x0 + c < a.W; c += 64) {
        uint32_t r[32];
        acc_ld32(sacc, co, c, r);
        const int xb = x0 + c;
        float v[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) v[e] = fmaxf(__uint_as_float(r[e]) + bias, 0.f);
        store_chunk_transposed<T>(stage, v, orow32 + (size_t)xb * a.out_stride, a.out_stride, a.W - xb, lane);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->acc_empty);
    }
  }
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_first_conv7x7s2(const void* x, const void* wpack, const float* bias, void* out, double* stats, int N, int H, int W,
                                           int relu, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && wpack && out, "first_conv7x7s2: null pointer");
  PFB_CHECK_ARG(dtype == PFB_F16 || dtype == PFB_BF16, "first_conv7x7s2: f16 / bf16 storage only (fp32 runs in cuDNN)");
  PFB_CHECK_ARG(N > 0 && H >= 2 && W >= 8 && H % 2 == 0 && W % 2 == 0, "first_conv7x7s2: bad shape %dx%dx%d (H, W even)", N, H, W);
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(wpack) & 15) == 0, "first_conv7x7s2: 16-byte alignment");
  cudaStream_t s = as_stream(stream);
  FcArgs a{};
  a.x = x; a.wpack = wpack; a.out = out; a.bias = bias; a.stats = stats;
  a.N = N; a.H = H; a.W = W; a.Ho = H / 2; a.Wo = W / 2;
  a.pairs = ceil_div(a.Ho, 2);
  a.nseg = ceil_div(a.Wo, kFcPix);
  a.n_items = N * a.pairs * a.nseg;
  int grid = sm_count();
  if (grid > a.n_items) grid = a.n_items;
  a.per_cta = ceil_div(a.n_items, grid);
  grid = ceil_div(a.n_items, a.per_cta);
  a.relu = relu;
  a.ab_fmt = dtype == PFB_F16 ? 0 : 1;
  const size_t smem = kFcABytes + kFcSlots * kFcSlotBytes + acc_tile_bytes(kFcPix) + 8 * 2048 + sizeof(FcBars) + 1024;
  ProfScope prof(KC_ENC_CONV1, s);  // encoder side: not part of the update-block conv roofline
  if (dtype == PFB_F16) {
    PFB_CUDA(cudaFuncSetAttribute(first_conv_umma_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PFB_CUDA(launch_pdl(first_conv_umma_kernel<__half>, dim3(grid), dim3(kFcThreads), smem, s, a));
  } else {
    PFB_CUDA(cudaFuncSetAttribute(first_conv_umma_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PFB_CUDA(launch_pdl(first_conv_umma_kernel<__nv_bfloat16>, dim3(grid), dim3(kFcThreads), smem, s, a));
  }
  return PFB_OK;
}

extern "C" PFB_API int pfb_flow_conv7x7(const float* flow, const void* wpack, const float* bias, void* out, int out_stride, int out_offset,
                                        int B, int H, int W, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(flow && wpack && out, "flow_conv7x7: null pointer");
  PFB_CHECK_ARG(dtype == PFB_F16 || dtype == PFB_BF16, "flow_conv7x7: f16 / bf16 storage only");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && out_stride >= out_offset + 128 && out_stride % 8 == 0 && out_offset % 8 == 0 &&
                    (reinterpret_cast<uintptr_t>(out) & 15) == 0,
                "flow_conv7x7: bad shape / alignment (out_stride, out_offset multiples of 8)");
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(flow) & 7) == 0 && (reinterpret_cast<uintptr_t>(wpack) & 15) == 0, "flow_conv7x7: alignment");
  cudaStream_t s = as_stream(stream);
  FlowConvArgs a{};
  a.flow = flow; a.wpack = wpack; a.bias = bias; a.out = out;
  a.B = B; a.H = H; a.W = W; a.out_stride = out_stride; a.out_offset = out_offset;
  a.nseg = ceil_div(W, kFcPix);
  a.n_items = B * H * a.nseg;
  int grid = sm_count();
  if (grid > a.n_items) grid = a.n_items;
  a.per_cta = ceil_div(a.n_items, grid);
  grid = ceil_div(a.n_items, a.per_cta);
  a.ab_fmt = dtype == PFB_F16 ? 0 : 1;
  const size_t smem = kFlABytes + 2 * kFlSlotBytes + acc_tile_bytes(kFcPix) + 8 * 2048 + sizeof(FlBars) + 1024;
  ProfScope prof(KC_FLOWCONV, s);
  if (dtype == PFB_F16) {
    PFB_CUDA(cudaFuncSetAttribute(flow_conv7x7_umma_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PFB_CUDA(launch_pdl(flow_conv7x7_umma_kernel<__half>, dim3(grid), dim3(kFlThreads), smem, s, a));
  } else {
    PFB_CUDA(cudaFuncSetAttribute(flow_conv7x7_umma_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PFB_CUDA(launch_pdl(flow_conv7x7_umma_kernel<__nv_bfloat16>, dim3(grid), dim3(kFlThreads), smem, s, a));
  }
  return PFB_OK;
}
