// Pieces shared by the wgmma correlation-volume kernels (csrc/corr_umma.cu, csrc/llaflow.cu): the MMA warpgroups' 128 x 128 patch
// GEMM, the accumulator hand-over to the epilogue warps, and the epilogue that writes one patch of the tiled pyramid.
#pragma once
#include <type_traits>

#include "umma.cuh"

namespace pfb {
using namespace sm90;

constexpr int kTileBytes = 128 * 128;  // 128 rows x 64 halves
constexpr int kCorrThreads = 13 * 32;

// The MMA warpgroups of the volume kernels: D[128 queries][128 targets] of one patch, rows 64 * wg .. 64 * wg + 63 per
// warpgroup, over `kchunks_here` 64-channel chunks at a_base / b_base (one 16 KB tile per chunk).
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

struct TiledOut {
  void* ptr[4];
  int h[4], w[4], tiles_x[4];
  unsigned map_elems[4];
};

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

// The epilogue of item i (target patch (ph, pw) of query block m_tile, sample b) of the tiled pyramid (layout: csrc/corr_tiled.cu),
// run by the 4 epilogue warps, thread <-> query `row`:
//   * level 0: the 128 x 128 accumulators times `scale`, staged as [2 tile rows][128 queries][128 bytes] (128-byte swizzle) and
//     written by one TMA bulk store through tmO, clipped at the map / N1 by the TMA unit;
//   * levels 1-3: means of the fp32 accumulators (one rounding per stored value), 16- / 8- / 4-byte stores; floor-sized 2 x 2
//     pooling, so a pooled cell never reads a target outside the map, and the pad columns of a level's last tile are written as 0.
// Targets of the patch outside the map (the last patch row / column) hold whatever the operands gave there: they land only in the
// level-0 pad cells of the last tiles, which the lookup masks (corr_tiled.cu), or are clipped by the TMA store.
// Waits for the MMA warpgroups' acc_full, releases acc_empty once the accumulators are read.  The caller waits for the last bulk
// store (tma_store_wait_read by row 0) before the CTA exits.
template <typename T>
__device__ __forceinline__ void tiled_epilogue_item(const float* sacc, uint8_t* sC, const CUtensorMap* tmO, const TiledOut& out, int row,
                                                    bool row_ok, T* o1, T* o2, T* o3, int i, int ph, int pw, int m_tile, int b,
                                                    float scale, uint64_t* acc_full, uint64_t* acc_empty) {
  const int lane = threadIdx.x & 31;
  const float s1 = 0.25f * scale, s2 = 0.0625f * scale, s3 = 0.015625f * scale;
  const bool leader = (row == 0);
  mbar_wait(acc_full, i & 1);
  float l2acc[4], l3acc[2];
#pragma unroll
  for (int c = 0; c < 4; ++c) {  // 32 accumulator columns = patch rows 2c, 2c+1 (16 columns each)
    uint32_t r[32];
    acc_ld32(sacc, row, c * 32, r);
    if (c == 0 && i > 0) {  // the previous bulk store must have drained the staging buffer
      if (leader) tma_store_wait_read();
      named_barrier_sync(1, 128);
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
        *reinterpret_cast<uint4*>(sC + (((rr >> 2) * 128 + row) * 128 + cidx * 16)) = u;
      }
    }
    // ---- pooled levels from the fp32 accumulators (one rounding per stored value) ----
    float l1[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      l1[j] = (__uint_as_float(r[2 * j]) + __uint_as_float(r[2 * j + 1])) + (__uint_as_float(r[16 + 2 * j]) + __uint_as_float(r[16 + 2 * j + 1]));
    if (o1 && row_ok) {
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
      if (o2 && row_ok) {
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
        if (o3 && row_ok) {
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
  if (lane == 0) mbar_arrive(acc_empty);
  fence_proxy_async();         // generic-proxy writes -> visible to the async (TMA) proxy
  named_barrier_sync(1, 128);  // the four epilogue warps
  if (leader) {
    // dims (element along the tile row, query, tile row, sample): clipped at the map / N1 by the TMA unit
    tma_store_4d(tmO, sC, pw * 64, m_tile * 128, ph * 2, b);
    tma_store_commit();
  }
}

// The level-0 store map of the tiled pyramid (box [2 tile rows][128 queries][128 bytes], 128-byte swizzle) and the per-level
// geometry, for N1 queries per sample against an H x W target grid.
int tiled_out_maps(void* const* pyr, int B, int N1, int H, int W, int L, pfb_dtype dt, TiledOut* out, CUtensorMap* tmO);

}  // namespace pfb
