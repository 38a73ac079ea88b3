// a1 + a2 on the Hopper tensor cores: all-pairs correlation as a TMA-fed wgmma GEMM whose epilogue
// also emits the 2x2 / 4x4 / 8x8 pooled pyramid levels, so the 4D volume is written once and never
// re-read (the reference does matmul -> divide -> 3x avg_pool2d, ptlflow/models/raft/corr.py:13-27,56-64).
//
//   D[n1, n2] = sum_c F1[b, n1, c] * F2[b, n2, c]        both operands K-major ("TN" GEMM)
//   M tile  = 128 consecutive query pixels n1 of one sample (TMA 3-D box over [B][N][C])
//   N tile  = an 8-row x 16-col patch of target pixels (TMA 4-D box over [B][H][W][C]): every pooled
//             level of that patch is an intra-thread reduction in the epilogue
//   K       = C (<= 256), whole-K tiles resident in shared memory, 128-byte swizzle
//
// CTA = 13 warps: 0-3 epilogue (thread = query row), 4-11 two MMA warpgroups (64 query rows each), 12 TMA producer.
// A (this CTA's 128 queries) is loaded once; B patches stream through a 1- or 2-deep ring (whatever fits next to the
// fp32 accumulator tile in shared memory); the MMA warpgroups hand each patch's accumulators over through that tile,
// so the epilogue of patch i overlaps the MMAs of patch i+1.
#include <stdlib.h>

#include <type_traits>

#include "umma.cuh"

namespace pfb {
using namespace sm90;

struct PyrOut {
  void* ptr[4];
};

constexpr int kTileBytes = 128 * 128;  // 128 rows x 64 halves
constexpr int kMaxKChunks = 4;

struct __align__(8) CorrBars {
  uint64_t a_full;
  uint64_t b_full[2];
  uint64_t b_empty[2];
  uint64_t acc_full;
  uint64_t acc_empty;
};

constexpr int kCorrThreads = 13 * 32;

// The MMA warpgroups of both volume kernels: D[128 queries][128 targets] of one patch, rows 64 * wg .. 64 * wg + 63 per
// warpgroup.  `stage_of(i, k)` gives the ring stage holding chunk k of item i; the ring slot is released per item
// (whole-K B stages, single_chunk = false) or per chunk (single_chunk = true).
template <bool BF16>
__device__ __forceinline__ void corr_mma_k(float (&d)[64], uint32_t a_base, uint32_t b_base, int kchunks_here, bool first) {
  const int wg = (threadIdx.x >> 7) - 1;
#pragma unroll 1
  for (int k = 0; k < kchunks_here; ++k) {
    const uint32_t al = gdesc_lo(a_base + k * kTileBytes + wg * 64 * 128, 16), bl = gdesc_lo(b_base + k * kTileBytes, 16);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
      wgmma<128, BF16>(d, gdesc(al + 2 * kk, kDescHiSw128), gdesc(bl + 2 * kk, kDescHiSw128), (first && k == 0 && kk == 0) ? 0u : 1u);
  }
}
__device__ __forceinline__ void corr_acc_handoff(float (&d)[64], float* sacc, uint64_t* acc_empty, uint64_t* acc_full, int i) {
  const int wg = (threadIdx.x >> 7) - 1;
  mbar_wait(acc_empty, (i & 1) ^ 1);
  acc_store<128>(sacc, d, wg * 64, threadIdx.x & 127);
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(acc_full);
}

template <typename T>
__device__ __forceinline__ float rt(float v) { return to_f32(from_f32<T>(v)); }

// store n consecutive values (already representable in T) at dst; `valid` of them are in range
template <typename T, int N>
__device__ __forceinline__ void store_row(T* dst, const float (&v)[N], int valid, bool vec_ok) {
  if (valid >= N && vec_ok) {
    if constexpr (N >= 8) {
#pragma unroll
      for (int q = 0; q < N / 8; ++q) {
        uint4 u;
        uint32_t* w = reinterpret_cast<uint32_t*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          T lo = from_f32<T>(v[q * 8 + 2 * e]), hi = from_f32<T>(v[q * 8 + 2 * e + 1]);
          w[e] = (uint32_t)(*reinterpret_cast<uint16_t*>(&lo)) | ((uint32_t)(*reinterpret_cast<uint16_t*>(&hi)) << 16);
        }
        reinterpret_cast<uint4*>(dst)[q] = u;
      }
    } else if constexpr (N == 4) {
      uint2 u;
      uint32_t* w = reinterpret_cast<uint32_t*>(&u);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        T lo = from_f32<T>(v[2 * e]), hi = from_f32<T>(v[2 * e + 1]);
        w[e] = (uint32_t)(*reinterpret_cast<uint16_t*>(&lo)) | ((uint32_t)(*reinterpret_cast<uint16_t*>(&hi)) << 16);
      }
      *reinterpret_cast<uint2*>(dst) = u;
    } else {
      T lo = from_f32<T>(v[0]), hi = from_f32<T>(v[1]);
      *reinterpret_cast<uint32_t*>(dst) =
          (uint32_t)(*reinterpret_cast<uint16_t*>(&lo)) | ((uint32_t)(*reinterpret_cast<uint16_t*>(&hi)) << 16);
    }
  } else {
#pragma unroll
    for (int e = 0; e < N; ++e)
      if (e < valid) dst[e] = from_f32<T>(v[e]);
  }
}

template <typename T>
__global__ void __launch_bounds__(kCorrThreads, 1)
corr_volume_umma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                        const __grid_constant__ CUtensorMap tmO, PyrOut out, int H, int W, int N, int kchunks, int levels,
                        float scale, int n_groups, int b_stages, int tma_store) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment for the 128B-swizzle atoms
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                     // kchunks tiles
  uint8_t* sB = smem + kchunks * kTileBytes;              // b_stages x kchunks tiles
  float* sacc = reinterpret_cast<float*>(sB + b_stages * kchunks * kTileBytes);  // fp32 accumulator tile, 128 columns
  // level-0 staging for the TMA store: [8 patch rows][128 queries][16 cols] (32 KB); a thread writes its query's
  // 32-byte row segments at (hh * 128 + row) * 32 -> consecutive lanes on consecutive segments, no bank conflicts
  uint8_t* sC = reinterpret_cast<uint8_t*>(sacc) + acc_tile_bytes(128);
  CorrBars* bars = reinterpret_cast<CorrBars*>(sC + (tma_store ? 8 * 128 * 32 : 0));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, group = blockIdx.y, b = blockIdx.z;
  const int PW = (W + 15) / 16, PH = (H + 7) / 8;
  const int n_tiles_total = PW * PH;
  const int my_tiles = (n_tiles_total - group + n_groups - 1) / n_groups;  // tiles group, group+n_groups, ...

  if (threadIdx.x == 0) {
    mbar_init(&bars->a_full, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bars->b_full[s], 1);
      mbar_init(&bars->b_empty[s], 8);  // one arrival per MMA warp
    }
    mbar_init(&bars->acc_full, 8);
    mbar_init(&bars->acc_empty, 4);  // one arrival per epilogue warp
    fence_barrier_init();
  }
  if (warp == 12 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (warp == 12) {
    // ================= TMA producer =================
    if (lane == 0) {
      mbar_arrive_expect_tx(&bars->a_full, kchunks * kTileBytes);
      for (int k = 0; k < kchunks; ++k) tma_load_3d(sA + k * kTileBytes, &tmA, &bars->a_full, k * 64, m_tile * 128, b);
      for (int i = 0; i < my_tiles; ++i) {
        const int s = i % b_stages, use = i / b_stages;
        const int tile = group + i * n_groups;
        const int ph = tile / PW, pw = tile - ph * PW;
        mbar_wait(&bars->b_empty[s], (use & 1) ^ 1);
        mbar_arrive_expect_tx(&bars->b_full[s], kchunks * kTileBytes);
        for (int k = 0; k < kchunks; ++k)
          tma_load_4d(sB + (s * kchunks + k) * kTileBytes, &tmB, &bars->b_full[s], k * 64, pw * 16, ph * 8, b);
      }
    }
  } else if (warp >= 4) {
    // ================= MMA warpgroups =================
    float d[64];
    mbar_wait(&bars->a_full, 0);
    for (int i = 0; i < my_tiles; ++i) {
      const int s = i % b_stages, use = i / b_stages;
      mbar_wait(&bars->b_full[s], use & 1);
      wgmma_fence();
      corr_mma_k<std::is_same<T, __nv_bfloat16>::value>(d, smem_u32(sA), smem_u32(sB + s * kchunks * kTileBytes), kchunks, true);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(d);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->b_empty[s]);  // smem stage free once these MMAs retired
      corr_acc_handoff(d, sacc, &bars->acc_empty, &bars->acc_full, i);
    }
  } else {
    // ================= epilogue (warps 0-3, 128 threads = 128 query rows) =================
    const int row = warp * 32 + lane;
    const int n1 = m_tile * 128 + row;
    const bool row_ok = n1 < N;
    const size_t q = (size_t)b * N + (row_ok ? n1 : 0);
    const int H1 = H >> 1, W1 = W >> 1, H2 = H >> 2, W2 = W >> 2, H3 = H >> 3, W3 = W >> 3;
    T* o0 = reinterpret_cast<T*>(out.ptr[0]) + q * (size_t)H * W;
    T* o1 = levels > 1 ? reinterpret_cast<T*>(out.ptr[1]) + q * (size_t)H1 * W1 : nullptr;
    T* o2 = levels > 2 ? reinterpret_cast<T*>(out.ptr[2]) + q * (size_t)H2 * W2 : nullptr;
    T* o3 = levels > 3 ? reinterpret_cast<T*>(out.ptr[3]) + q * (size_t)H3 * W3 : nullptr;
    // vector stores need every row start 16-byte (level 0/1), 8-byte (2), 4-byte (3) aligned
    const bool vec0 = (W % 8) == 0, vec1 = (W1 % 8) == 0, vec2 = (W2 % 4) == 0, vec3 = (W3 % 2) == 0;
    for (int i = 0; i < my_tiles; ++i) {
      const int tile = group + i * n_groups;
      const int ph = tile / PW, pw = tile - ph * PW;
      mbar_wait(&bars->acc_full, i & 1);
      if (tma_store && i > 0) {  // the previous tile's bulk store must have drained the staging buffer
        if (threadIdx.x == 0) tma_store_wait_read();
        named_barrier_sync(1, 128);
      }
      float l1prev[8], l2prev[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {  // 32 columns = patch rows 2c, 2c+1
        uint32_t r[32];
        acc_ld32(sacc, row, c * 32, r);
        float v[2][16];
#pragma unroll
        for (int e = 0; e < 32; ++e) v[e >> 4][e & 15] = rt<T>(__uint_as_float(r[e]) * scale);
        if (tma_store) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) store_row<T, 16>(reinterpret_cast<T*>(sC + ((2 * c + rr) * 128 + row) * 32), v[rr], 16, true);
        } else if (row_ok) {
#pragma unroll
          for (int rr = 0; rr < 2; ++rr) {
            const int h2 = ph * 8 + 2 * c + rr, w2 = pw * 16;
            if (h2 < H) store_row<T, 16>(o0 + (size_t)h2 * W + w2, v[rr], W - w2, vec0);
          }
        }
        float l1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) l1[j] = rt<T>(0.25f * (v[0][2 * j] + v[0][2 * j + 1] + v[1][2 * j] + v[1][2 * j + 1]));
        if (row_ok && o1) {
          const int i1 = ph * 4 + c, j1 = pw * 8;
          if (i1 < H1) store_row<T, 8>(o1 + (size_t)i1 * W1 + j1, l1, W1 - j1, vec1);
        }
        if ((c & 1) == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) l1prev[j] = l1[j];
        } else {
          float l2[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) l2[j] = rt<T>(0.25f * (l1prev[2 * j] + l1prev[2 * j + 1] + l1[2 * j] + l1[2 * j + 1]));
          if (row_ok && o2) {
            const int i2 = ph * 2 + (c >> 1), j2 = pw * 4;
            if (i2 < H2) store_row<T, 4>(o2 + (size_t)i2 * W2 + j2, l2, W2 - j2, vec2);
          }
          if (c == 1) {
#pragma unroll
            for (int j = 0; j < 4; ++j) l2prev[j] = l2[j];
          } else {
            float l3[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) l3[j] = rt<T>(0.25f * (l2prev[2 * j] + l2prev[2 * j + 1] + l2[2 * j] + l2[2 * j + 1]));
            if (row_ok && o3) {
              const int i3 = ph, j3 = pw * 2;
              if (i3 < H3) store_row<T, 2>(o3 + (size_t)i3 * W3 + j3, l3, W3 - j3, vec3);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->acc_empty);
      if (tma_store) {
        fence_proxy_async();         // generic-proxy writes -> visible to the async (TMA) proxy
        named_barrier_sync(1, 128);  // the four epilogue warps
        if (threadIdx.x == 0) {
          tma_store_4d(&tmO, sC, pw * 16, m_tile * 128, ph * 8, b);  // clipped at W / N / H by the TMA unit
          tma_store_commit();
        }
      }
    }
    if (tma_store && threadIdx.x == 0) tma_store_wait_read();
  }
}

// =====================================================================================================================
// Tiled-pyramid variant (round 2): same GEMM, output in the T84 layout of csrc/corr_tiled.cu (4 x 8 tiles of 64 bytes).
//
//   * one target patch per item (N = 128): the MMA warpgroups of the kernel above, accumulators handed over through the
//     shared-memory tile; 4 epilogue warps, thread <-> query row.
//   * pooled levels are means of the fp32 accumulators, rounded once (closer to the fp32 reference than re-rounding
//     every level like the reference's half path does; also 2 conversions fewer per element), packed conversions.
//   * level 0 leaves through one TMA bulk store per patch: box [2 tile rows][128 queries][128 bytes] (the two tiles a
//     patch owns in a tile row are contiguous), 128-byte swizzled staging; level 1 is one full 64-byte tile per
//     (query, patch) written with 16-byte stores.
//   B operand ring: 3 stages of one 64-channel chunk of the patch (16 KB).  One CTA per SM.
struct __align__(8) CorrTBars {
  uint64_t a_full;
  uint64_t b_full[3];
  uint64_t b_empty[3];
  uint64_t acc_full;
  uint64_t acc_empty;
};

struct TiledOut {
  void* ptr[4];
  int h[4], w[4], tiles_x[4];
  unsigned map_elems[4];
};

__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
               : "memory");
}

template <typename T>
__device__ __forceinline__ uint32_t cvt_pack2(float lo, float hi);
template <>
__device__ __forceinline__ uint32_t cvt_pack2<__half>(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <>
__device__ __forceinline__ uint32_t cvt_pack2<__nv_bfloat16>(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <typename T>
__global__ void __launch_bounds__(kCorrThreads, 1)
corr_volume_tiled_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                         const __grid_constant__ CUtensorMap tmO, TiledOut out, int H, int W, int N1, int kchunks, int levels,
                         float scale, int ab_fmt) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                   // kchunks x 16 KB
  uint8_t* sB = sA + kchunks * kTileBytes;              // 3 stages x 16 KB
  float* sacc = reinterpret_cast<float*>(sB + 3 * kTileBytes);  // fp32 accumulator tile, 128 columns
  uint8_t* sC = reinterpret_cast<uint8_t*>(sacc) + acc_tile_bytes(128);  // 32 KB: [tile row 2][chunk 8][query 128][16 B]
  CorrTBars* bars = reinterpret_cast<CorrTBars*>(sC + 2 * kTileBytes);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, b = blockIdx.z;
  const int PW = (W + 15) / 16, PH = (H + 7) / 8;
  const int n_patches = PW * PH;
  const int n_items = n_patches;

  if (threadIdx.x == 0) {
    mbar_init(&bars->a_full, 1);
    for (int s = 0; s < 3; ++s) {
      mbar_init(&bars->b_full[s], 1);
      mbar_init(&bars->b_empty[s], 8);  // one arrival per MMA warp
    }
    mbar_init(&bars->acc_full, 8);
    mbar_init(&bars->acc_empty, 4);  // one arrival per epilogue warp
    fence_barrier_init();
  }
  if (warp == 12 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    prefetch_tmap(&tmO);
  }
  __syncthreads();

  if (warp == 12) {
    // ================= TMA producer =================
    if (lane == 0) {
      mbar_arrive_expect_tx(&bars->a_full, kchunks * kTileBytes);
      for (int k = 0; k < kchunks; ++k) tma_load_3d(sA + k * kTileBytes, &tmA, &bars->a_full, k * 64, m_tile * 128, b);
      int st = 0;
      uint32_t phs = 0;
      for (int i = 0; i < n_items; ++i) {
        const int ph0 = i / PW, pw0 = i - ph0 * PW;
        for (int k = 0; k < kchunks; ++k) {
          mbar_wait(&bars->b_empty[st], phs ^ 1);
          mbar_arrive_expect_tx(&bars->b_full[st], kTileBytes);
          tma_load_4d(sB + st * kTileBytes, &tmB, &bars->b_full[st], k * 64, pw0 * 16, ph0 * 8, b);
          if (++st == 3) { st = 0; phs ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ================= MMA warpgroups =================
    float d[64];
    mbar_wait(&bars->a_full, 0);
    int st = 0;
    uint32_t phs = 0;
    for (int i = 0; i < n_items; ++i) {
      for (int k = 0; k < kchunks; ++k) {
        mbar_wait(&bars->b_full[st], phs);
        wgmma_fence();
        corr_mma_k<std::is_same<T, __nv_bfloat16>::value>(d, smem_u32(sA + k * kTileBytes), smem_u32(sB + st * kTileBytes), 1, k == 0);
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(d);
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->b_empty[st]);
        if (++st == 3) { st = 0; phs ^= 1; }
      }
      corr_acc_handoff(d, sacc, &bars->acc_empty, &bars->acc_full, i);
    }
  } else {
    // ================= epilogue: 4 warps, thread <-> query row =================
    const int quarter = warp & 3, grp = 0;
    const int row = quarter * 32 + lane;
    const int n1 = m_tile * 128 + row;
    const bool row_ok = n1 < N1;
    const size_t q = (size_t)b * N1 + (row_ok ? n1 : 0);
    uint8_t* sCg = sC;
    T* o1 = levels > 1 ? reinterpret_cast<T*>(out.ptr[1]) + q * out.map_elems[1] : nullptr;
    T* o2 = levels > 2 ? reinterpret_cast<T*>(out.ptr[2]) + q * out.map_elems[2] : nullptr;
    T* o3 = levels > 3 ? reinterpret_cast<T*>(out.ptr[3]) + q * out.map_elems[3] : nullptr;
    const float s1 = 0.25f * scale, s2 = 0.0625f * scale, s3 = 0.015625f * scale;
    const bool leader = (row == 0);
    for (int i = 0; i < n_items; ++i) {
      const int p = i;
      const bool p_ok = p < n_patches;
      const int ph = p / PW, pw = p - ph * PW;
      mbar_wait(&bars->acc_full, i & 1);
      float l2acc[4], l3acc[2];
#pragma unroll
      for (int c = 0; c < 4; ++c) {  // 32 accumulator columns = patch rows 2c, 2c+1 (16 columns each)
        uint32_t r[32];
        acc_ld32(sacc, row, c * 32, r);
        if (c == 0 && i > 0) {  // the previous bulk store of this group must have drained the staging buffer
          if (leader) tma_store_wait_read();
          named_barrier_sync(1 + grp, 128);
        }
        // ---- level 0: scale, pack, stage.  patch row rr -> tile row rr >> 2, row-in-tile rr & 3; columns 0-7 / 8-15 -> tile column 0 / 1
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int rr = 2 * c + e;
#pragma unroll
          for (int txh = 0; txh < 2; ++txh) {
            uint4 u;
            u.x = cvt_pack2<T>(__uint_as_float(r[e * 16 + txh * 8 + 0]) * scale, __uint_as_float(r[e * 16 + txh * 8 + 1]) * scale);
            u.y = cvt_pack2<T>(__uint_as_float(r[e * 16 + txh * 8 + 2]) * scale, __uint_as_float(r[e * 16 + txh * 8 + 3]) * scale);
            u.z = cvt_pack2<T>(__uint_as_float(r[e * 16 + txh * 8 + 4]) * scale, __uint_as_float(r[e * 16 + txh * 8 + 5]) * scale);
            u.w = cvt_pack2<T>(__uint_as_float(r[e * 16 + txh * 8 + 6]) * scale, __uint_as_float(r[e * 16 + txh * 8 + 7]) * scale);
            // staging = TMA box [tile row 2][query 128][128 bytes = the two tiles of that tile row], 128-byte swizzle:
            // 16-byte chunk (tile column txh, row-in-tile rr & 3) of query `row` sits at chunk index ^ (row & 7)
            const int cidx = (txh * 4 + (rr & 3)) ^ (row & 7);
            *reinterpret_cast<uint4*>(sCg + (((rr >> 2) * 128 + row) * 128 + cidx * 16)) = u;
          }
        }
        // ---- pooled levels from the fp32 accumulators (one rounding per stored value) ----
        float l1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
          l1[j] = (__uint_as_float(r[2 * j]) + __uint_as_float(r[2 * j + 1])) + (__uint_as_float(r[16 + 2 * j]) + __uint_as_float(r[16 + 2 * j + 1]));
        if (o1 && row_ok && p_ok) {
          const int i1 = ph * 4 + c, j1 = pw * 8;
          if (i1 < out.h[1] && j1 < out.w[1]) {
            const int valid = out.w[1] - j1;  // columns of this tile inside the map; the rest are pad columns = 0
            uint4 u;
            u.x = cvt_pack2<T>(valid > 0 ? l1[0] * s1 : 0.f, valid > 1 ? l1[1] * s1 : 0.f);
            u.y = cvt_pack2<T>(valid > 2 ? l1[2] * s1 : 0.f, valid > 3 ? l1[3] * s1 : 0.f);
            u.z = cvt_pack2<T>(valid > 4 ? l1[4] * s1 : 0.f, valid > 5 ? l1[5] * s1 : 0.f);
            u.w = cvt_pack2<T>(valid > 6 ? l1[6] * s1 : 0.f, valid > 7 ? l1[7] * s1 : 0.f);
            *reinterpret_cast<uint4*>(o1 + (size_t)(ph * out.tiles_x[1] + pw) * 32 + c * 8) = u;
          }
        }
        if ((c & 1) == 0) {
#pragma unroll
          for (int j = 0; j < 4; ++j) l2acc[j] = l1[2 * j] + l1[2 * j + 1];
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) l2acc[j] += l1[2 * j] + l1[2 * j + 1];
          if (o2 && row_ok && p_ok) {
            const int i2 = ph * 2 + (c >> 1), j2 = pw * 4;
            if (i2 < out.h[2] && j2 < out.w[2]) {
              const int valid = out.w[2] - j2;
              uint2 u;
              u.x = cvt_pack2<T>(valid > 0 ? l2acc[0] * s2 : 0.f, valid > 1 ? l2acc[1] * s2 : 0.f);
              u.y = cvt_pack2<T>(valid > 2 ? l2acc[2] * s2 : 0.f, valid > 3 ? l2acc[3] * s2 : 0.f);
              *reinterpret_cast<uint2*>(o2 + (size_t)((i2 >> 2) * out.tiles_x[2] + (pw >> 1)) * 32 + (i2 & 3) * 8 + (pw & 1) * 4) = u;
            }
          }
          if (c == 1) {
            l3acc[0] = l2acc[0] + l2acc[1];
            l3acc[1] = l2acc[2] + l2acc[3];
          } else {
            l3acc[0] += l2acc[0] + l2acc[1];
            l3acc[1] += l2acc[2] + l2acc[3];
            if (o3 && row_ok && p_ok) {
              const int i3 = ph, j3 = pw * 2;
              if (i3 < out.h[3] && j3 < out.w[3]) {
                const int valid = out.w[3] - j3;
                const uint32_t u = cvt_pack2<T>(l3acc[0] * s3, valid > 1 ? l3acc[1] * s3 : 0.f);
                *reinterpret_cast<uint32_t*>(o3 + (size_t)((i3 >> 2) * out.tiles_x[3] + (pw >> 2)) * 32 + (i3 & 3) * 8 + (pw & 3) * 2) = u;
              }
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->acc_empty);
      fence_proxy_async();               // generic-proxy writes -> visible to the async (TMA) proxy
      named_barrier_sync(1 + grp, 128);  // the four warps of this group
      if (leader && p_ok) {
        // dims (element along the tile row, query, tile row, sample): clipped at the map / N1 by the TMA unit
        tma_store_4d(&tmO, sCg, pw * 64, m_tile * 128, ph * 2, b);
        tma_store_commit();
      }
    }
    if (leader) tma_store_wait_read();
  }
}

bool corr_volume_umma_supported(int B, int H, int W, int C, int L, pfb_dtype dt) {
  if (dt != PFB_F16 && dt != PFB_BF16) return false;
  if (C % 64 != 0 || C > 64 * kMaxKChunks) return false;
  if (L < 1 || L > 4) return false;
  if (H < 1 || W < 1 || B < 1 || B > 65535) return false;
  return true;
}

int corr_volume_umma(const void* f1, const void* f2, void* const* pyr, int B, int N1, int H, int W, int C, int L, float scale,
                     pfb_dtype dt, cudaStream_t s) {
  const int N = N1;  // queries; targets are the H x W grid (equal to the query grid for RAFT, its own for SEA-RAFT levels)
  const int kchunks = C / 64;
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)N, (uint64_t)B};
    uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)N * C * 2};
    uint32_t box[3] = {64, 128, 1};
    int rc = make_tensor_map(&tmA, f1, dt, 3, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {64, 16, 8, 1};
    int rc = make_tensor_map(&tmB, f2, dt, 4, dims, str, box);
    if (rc) return rc;
  }
  PyrOut out{};
  for (int l = 0; l < L; ++l) out.ptr[l] = pyr[l];
  // level 0 leaves through TMA bulk stores (full-sector writes issued by the copy engine instead of 16-byte
  // per-thread stores to 128 different query maps); needs 16-byte aligned target rows
  static const int env_tma = getenv("PFB_VOLUME_TMA_STORE") ? atoi(getenv("PFB_VOLUME_TMA_STORE")) : 1;
  // shared memory: A (kchunks tiles) + accumulator tile + B ring (2 stages where they fit, else 1) + level-0 staging where
  // it fits
  const size_t smem_cap = 227 * 1024 - sizeof(CorrBars) - 1024;
  const size_t fixed = (size_t)kchunks * kTileBytes + acc_tile_bytes(128), stage = (size_t)kchunks * kTileBytes, staging = 8 * 128 * 32;
  int tma_store = (env_tma && (W % 8) == 0) ? 1 : 0;
  if (fixed + stage + (tma_store ? staging : 0) > smem_cap) tma_store = 0;
  const int b_stages = fixed + 2 * stage + (tma_store ? staging : 0) <= smem_cap ? 2 : 1;
  CUtensorMap tmO = tmA;
  if (tma_store) {
    // dims ordered (w, query, h, b) so that the shared-memory box is [h][query][w]
    uint64_t dims[4] = {(uint64_t)W, (uint64_t)N, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)H * W * 2, (uint64_t)W * 2, (uint64_t)N * H * W * 2};
    uint32_t box[4] = {16, 128, 8, 1};
    int rc = make_tensor_map_linear(&tmO, pyr[0], dt, 4, dims, str, box);
    if (rc) return rc;
  }
  const int m_tiles = ceil_div(N, 128);
  const int n_tiles = ceil_div(W, 16) * ceil_div(H, 8);
  // enough CTAs for ~2 waves of the machine; each CTA keeps its A tile and walks its share of patches
  int groups = ceil_div(2 * sm_count(), m_tiles * B);
  if (groups < 1) groups = 1;
  if (groups > n_tiles) groups = n_tiles;
  const size_t smem = fixed + b_stages * stage + (tma_store ? staging : 0) + sizeof(CorrBars) + 1024;
  dim3 grid(m_tiles, groups, B);
  ProfScope prof(KC_VOLUME, s);
  if (dt == PFB_F16) {
    PFB_CUDA(cudaFuncSetAttribute(corr_volume_umma_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    corr_volume_umma_kernel<__half><<<grid, kCorrThreads, smem, s>>>(tmA, tmB, tmO, out, H, W, N, kchunks, L, scale, groups, b_stages, tma_store);
  } else {
    PFB_CUDA(cudaFuncSetAttribute(corr_volume_umma_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    corr_volume_umma_kernel<__nv_bfloat16><<<grid, kCorrThreads, smem, s>>>(tmA, tmB, tmO, out, H, W, N, kchunks, L, scale, groups, b_stages, tma_store);
  }
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

namespace pfb {

bool corr_volume_tiled_supported(int B, int H, int W, int C, int L, pfb_dtype dt) {
  if (dt != PFB_F16 && dt != PFB_BF16) return false;
  if (C % 64 != 0 || C > 64 * kMaxKChunks) return false;
  if (L < 1 || L > 4) return false;
  if (H < 1 || W < 1 || B < 1 || B > 65535) return false;
  return true;
}

int corr_volume_tiled(const void* f1, const void* f2, void* const* pyr, int B, int N1, int H, int W, int C, int L, float scale,
                      pfb_dtype dt, cudaStream_t s) {
  const int kchunks = C / 64;
  CUtensorMap tmA, tmB, tmO;
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)N1, (uint64_t)B};
    uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)N1 * C * 2};
    uint32_t box[3] = {64, 128, 1};
    int rc = make_tensor_map(&tmA, f1, dt, 3, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {64, 16, 8, 1};
    int rc = make_tensor_map(&tmB, f2, dt, 4, dims, str, box);
    if (rc) return rc;
  }
  TiledOut out{};
  for (int l = 0; l < L; ++l) {
    out.ptr[l] = pyr[l];
    out.h[l] = H >> l;
    out.w[l] = W >> l;
    out.tiles_x[l] = (out.w[l] + 7) >> 3;
    out.map_elems[l] = (unsigned)(((out.h[l] + 3) >> 2) * out.tiles_x[l] * 32);
  }
  {
    // level-0 store map: a tile row of a query's map is tiles_x * 64 contiguous bytes, so the two tiles a patch owns in one
    // tile row are ONE 128-byte run: box = [2 tile rows][128 queries][128 bytes], swizzled like an operand tile so that
    // the per-thread 16-byte staging stores are conflict-free.  (The first version used 16-byte inner rows -- 2048 TMA
    // requests per 32 KB box -- and ran at 1.56 TB/s; ncu r02b.)
    const uint64_t tx0 = (uint64_t)out.tiles_x[0], ty0 = (uint64_t)((H + 3) >> 2), map_bytes = ty0 * tx0 * 64;
    uint64_t dims[4] = {32 * tx0, (uint64_t)N1, ty0, (uint64_t)B};
    uint64_t str[3] = {map_bytes, 64 * tx0, (uint64_t)N1 * map_bytes};
    uint32_t box[4] = {64, 128, 2, 1};
    int rc = make_tensor_map(&tmO, pyr[0], dt, 4, dims, str, box);
    if (rc) return rc;
  }
  const int m_tiles = ceil_div(N1, 128);
  const size_t smem = (size_t)kchunks * kTileBytes + 3 * kTileBytes + acc_tile_bytes(128) + 2 * kTileBytes + sizeof(CorrTBars) + 1024;
  dim3 grid(m_tiles, 1, B);
  ProfScope prof(KC_VOLUME, s);
  if (dt == PFB_F16) {
    PFB_CUDA(cudaFuncSetAttribute(corr_volume_tiled_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    corr_volume_tiled_kernel<__half><<<grid, kCorrThreads, smem, s>>>(tmA, tmB, tmO, out, H, W, N1, kchunks, L, scale, 0);
  } else {
    PFB_CUDA(cudaFuncSetAttribute(corr_volume_tiled_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    corr_volume_tiled_kernel<__nv_bfloat16><<<grid, kCorrThreads, smem, s>>>(tmA, tmB, tmO, out, H, W, N1, kchunks, L, scale, 1);
  }
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

extern "C" PFB_API int pfb_corr_volume_build_tiled(const void* fmap1, const void* fmap2, void* const* pyramid, int B, int H1, int W1,
                                                   int H2, int W2, int C, int levels, float scale, pfb_dtype dtype, pfb_stream stream) {
  using namespace pfb;
  PFB_CHECK_ARG(fmap1 && fmap2 && pyramid, "corr_volume_build_tiled: null pointer");
  PFB_CHECK_ARG(B > 0 && H1 > 0 && W1 > 0 && H2 > 0 && W2 > 0 && C > 0, "corr_volume_build_tiled: bad shape");
  PFB_CHECK_ARG(levels >= 1 && levels <= 4 && (H2 >> (levels - 1)) >= 1 && (W2 >> (levels - 1)) >= 1,
                "corr_volume_build_tiled: %dx%d target grid cannot hold %d levels (1..4)", H2, W2, levels);
  for (int l = 0; l < levels; ++l)
    PFB_CHECK_ARG(pyramid[l] && (reinterpret_cast<uintptr_t>(pyramid[l]) & 15) == 0, "corr_volume_build_tiled: pyramid[%d] null or not 16-byte aligned", l);
  if (!corr_volume_tiled_supported(B, H2, W2, C, levels, dtype)) {
    set_error("corr_volume_build_tiled: needs f16/bf16 storage and C a multiple of 64, <= 256 (C=%d dtype=%d)", C, (int)dtype);
    return PFB_ERR_UNSUPPORTED;
  }
  return corr_volume_tiled(fmap1, fmap2, pyramid, B, H1 * W1, H2, W2, C, levels, scale, dtype, as_stream(stream));
}
