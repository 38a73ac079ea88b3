// a4 on the tensor cores: on-the-fly correlation + lookup without the 4D volume (f16 / bf16, radius 4, C % 64 == 0, C <= 256).
//
// Replaces, for those shapes, the reference's alt_cuda_corr kernel (ptlflow/utils/external/alt_cuda_corr/
// correlation_kernel.cu:18-119: one warp per 4x8 query tile, 32-channel chunks, scalar FMAs, global RMW per tap) and this
// library's own SIMT kernel (csrc/corr.cu: one warp per query, a 256-long dot product per window tap from L2).
//
// Work item = (tile of 8 x 16 neighbouring queries, pyramid level).  The windows of neighbouring queries overlap almost
// completely when the flow is locally smooth, so the item multiplies the tile's 128 query vectors with a REGION of the
// level's feature map that contains all their windows -- anchored at the tile's smallest window origin, 32 targets wide, in
// bands of 8 rows (band stride 7, so that every vertical tap pair lies inside one band):
//     D[128 queries][256 targets] = F1_tile[128][C] . F2_band[256][C]^T        (wgmma: two warpgroups of m64n128 per band half)
// Both operands are TMA boxes of the pixel-major feature maps (out-of-map targets are zero-filled by the TMA unit: the
// zero padding of raft/utils.py:71-75 for free).  The MMA warpgroups dump the accumulator rows, scaled, to shared memory
// (storage type -- the same rounding the materialised volume has); each epilogue thread owns one query and blends the window rows that
// fall into this band (x-major order of corr.py:43-47) and stages the level's 81 outputs for a coalesced store.
// Queries whose window does not fit the region (rough flow inside a tile) are flagged and recomputed by the SIMT kernel
// (exact same values, one warp per flagged query), so the result never depends on the smoothness of the flow.
#include <stdlib.h>

#include <algorithm>
#include <vector>
#include <stdio.h>
#include <type_traits>

#include "umma.cuh"

namespace pfb {
using namespace sm90;

constexpr int kOtfTileBytes = 128 * 128;       // 128 rows x 64 channels
constexpr int kOtfMaxBands = 8;                // 7 * 8 + 1 = 57 region rows at most
constexpr int kOtfRW = 32;
constexpr int kOtfDumpPitch = 520;             // bytes per accumulator-dump row: 256 targets x 2 bytes + 8 (130 words: 8-byte stores of a
                                               // half-warp and the gather's 4-byte loads of a warp spread over the banks)
constexpr int kOtfMaxStages = 6;               // B-operand ring: 64-channel chunks of one band half (4 rows x 32 columns, 16 KB each)

struct OtfArgs {
  const float* coords;
  void* out;
  unsigned char* flags;  // [B*H*W]: set to 1 for queries the region could not serve (recomputed by the SIMT kernel)
  int B, H, W, kchunks, levels, out_stride;
  int lh[4], lw[4];
  float scale;
  int tiles_x, tiles_y, n_tiles;
  int b_stages;
  unsigned long long* trace;  // PFB_OTF_TRACE: [CTA][64] clock64 stamps of the CTA's second work item (phase timeline), else null
};

struct __align__(8) OtfBars {
  uint64_t a_full, a_empty;
  uint64_t b_full[kOtfMaxStages], b_empty[kOtfMaxStages];
  uint64_t dump_full, dump_empty;
  uint64_t reg_full[2], reg_empty[2];
  int region[2][4];  // per item parity: bx0, by0, number of bands
  int red[4][3];
};

template <typename T>
__device__ __forceinline__ uint32_t otf_pack2(float lo, float hi);
template <>
__device__ __forceinline__ uint32_t otf_pack2<__half>(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <>
__device__ __forceinline__ uint32_t otf_pack2<__nv_bfloat16>(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <typename T>
__device__ __forceinline__ float otf_bits_to_f32(unsigned short b);
template <>
__device__ __forceinline__ float otf_bits_to_f32<__half>(unsigned short b) { return __half2float(__ushort_as_half(b)); }
template <>
__device__ __forceinline__ float otf_bits_to_f32<__nv_bfloat16>(unsigned short b) { return __uint_as_float((unsigned)b << 16); }
template <typename T>
__device__ __forceinline__ unsigned short otf_f32_to_bits(float v);
template <>
__device__ __forceinline__ unsigned short otf_f32_to_bits<__half>(float v) { return __half_as_ushort(__float2half_rn(v)); }
template <>
__device__ __forceinline__ unsigned short otf_f32_to_bits<__nv_bfloat16>(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }

// Roles: warps 0-7 = epilogue (two threads per query of the tile: warps w and w + 4 hold the same queries and split the
// window rows), warps 8-15 = two MMA warpgroups (query halves; the band's two target halves one after the other),
// warp 16 = TMA producer.  The three
// walk the same list of work items (tile, level) and are coupled only through mbarriers:
//   reg_full / reg_empty [item parity]  the epilogue publishes the item's region (anchor, bands) one item AHEAD, so the
//                                       producer streams the next item's operands while the epilogue still blends this one
//   a_full / a_empty                    the tile's query vectors (kchunks x 16 KB), loaded once per item
//   b_full / b_empty [stage]            ring of 64-channel chunks of a band half (16 KB each): consumed once,
//                                       so the band is never resident as a whole
//   dump_full / dump_empty              the band's accumulator dump: band k+1 is multiplied (into registers) while the
//                                       epilogue blends band k out of the dump
constexpr int kOtfThreads = 17 * 32;
template <typename T, int R>
__global__ void __launch_bounds__(kOtfThreads, 1)
corr_onthefly_umma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB0,
                          const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmB2,
                          const __grid_constant__ CUtensorMap tmB3, const OtfArgs a) {
  constexpr int D = 2 * R + 2, K = 2 * R + 1, KK = K * K;
  constexpr int SP = KK + 1;  // staging row pitch in halfs (odd number of 32-bit words: conflict-free per-thread rows)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;                                       // kchunks x 16 KB
  uint8_t* sB = sA + a.kchunks * kOtfTileBytes;             // b_stages x 16 KB
  uint8_t* sD = sB + a.b_stages * kOtfTileBytes;            // accumulator dump [128 queries][256 targets] (storage type), pitch 520 B
  unsigned short* sOut = reinterpret_cast<unsigned short*>(sD + 128 * kOtfDumpPitch);  // [128][SP] staged outputs of one level
  OtfBars* bars = reinterpret_cast<OtfBars*>(reinterpret_cast<uint8_t*>(sOut) + ((128 * SP * 2 + 15) & ~15));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(&bars->a_full, 1);
    mbar_init(&bars->a_empty, 8);  // one arrival per MMA warp
    for (int s = 0; s < kOtfMaxStages; ++s) {
      mbar_init(&bars->b_full[s], 1);
      mbar_init(&bars->b_empty[s], 8);
    }
    mbar_init(&bars->dump_full, 8);  // one arrival per MMA warp
    mbar_init(&bars->dump_empty, 8);  // one arrival per epilogue warp
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bars->reg_full[s], 1);
      mbar_init(&bars->reg_empty[s], 9);  // producer + the 8 MMA warps have read the slot
    }
    fence_barrier_init();
  }
  if (warp == 16 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB0);
  }
  __syncthreads();
  const int n_items = a.n_tiles * a.levels;
#define OTF_TR(slot) do { if (a.trace && n == 1 && (slot) < 64) a.trace[blockIdx.x * 64 + (slot)] = clock64(); } while (0)

  if (warp == 16) {
    // ================= TMA producer =================
    if (lane == 0) {
      int sb = 0;
      uint32_t phb = 0;
      int n = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++n) {
        const int slot = n & 1;
        mbar_wait(&bars->reg_full[slot], (n >> 1) & 1);
        const int bx0 = bars->region[slot][0], by0 = bars->region[slot][1], nb = bars->region[slot][2];
        mbar_arrive(&bars->reg_empty[slot]);
        const int tile = item / a.levels, l = item - tile * a.levels;
        const int tx = tile % a.tiles_x, ty = (tile / a.tiles_x) % a.tiles_y, b = tile / (a.tiles_x * a.tiles_y);
        const CUtensorMap* tmB = l == 0 ? &tmB0 : (l == 1 ? &tmB1 : (l == 2 ? &tmB2 : &tmB3));
        mbar_wait(&bars->a_empty, (n & 1) ^ 1);  // the previous item's MMAs are done with the query tile
        mbar_arrive_expect_tx(&bars->a_full, a.kchunks * kOtfTileBytes);
        for (int k = 0; k < a.kchunks; ++k) tma_load_4d(sA + k * kOtfTileBytes, &tmA, &bars->a_full, k * 64, tx * 16, ty * 8, b);
        for (int kb = 0; kb < nb; ++kb) {
          OTF_TR(8 + kb * 6 + 0);
          for (int nh = 0; nh < 2; ++nh) {
            for (int k = 0; k < a.kchunks; ++k) {
              mbar_wait(&bars->b_empty[sb], phb ^ 1);
              mbar_arrive_expect_tx(&bars->b_full[sb], kOtfTileBytes);
              tma_load_4d(sB + sb * kOtfTileBytes, tmB, &bars->b_full[sb], k * 64, bx0, by0 + 7 * kb + 4 * nh, b);
              if (++sb == a.b_stages) { sb = 0; phb ^= 1; }
            }
          }
        }
      }
    }
  } else if (warp >= 8) {
    // ================= MMA warpgroups: query half mh, m64n128 per target half nh of the band =================
    const int mh = (threadIdx.x >> 7) - 2, tid = threadIdx.x & 127;
    float d[64];
    int sb = 0, g = 0;
    uint32_t phb = 0;
    int n = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++n) {
      const int slot = n & 1;
      mbar_wait(&bars->reg_full[slot], (n >> 1) & 1);
      const int nb = bars->region[slot][2];
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->reg_empty[slot]);
      mbar_wait(&bars->a_full, n & 1);
      for (int kb = 0; kb < nb; ++kb, ++g) {
       for (int nh = 0; nh < 2; ++nh) {
        for (int k = 0; k < a.kchunks; ++k) {
          mbar_wait(&bars->b_full[sb], phb);
          const uint32_t al = gdesc_lo(smem_u32(sA + k * kOtfTileBytes) + mh * 64 * 128, 16);
          const uint32_t bl = gdesc_lo(smem_u32(sB + sb * kOtfTileBytes), 16);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            wgmma<128, std::is_same<T, __nv_bfloat16>::value>(d, gdesc(al + 2 * kk, kDescHiSw128), gdesc(bl + 2 * kk, kDescHiSw128), (k | kk) != 0);
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(d);
          __syncwarp();
          if (lane == 0) mbar_arrive(&bars->b_empty[sb]);
          if (++sb == a.b_stages) { sb = 0; phb ^= 1; }
        }
        if (threadIdx.x == 256) OTF_TR(8 + kb * 6 + 1);
        // ---- accumulator -> dump rows: scaled, then rounded to the storage type (the materialised volume's rounding).
        // Scaling first keeps f16 finite where |a.b| exceeds 65504 but the scaled correlation does not ----
        if (nh == 0) mbar_wait(&bars->dump_empty, (g & 1) ^ 1);  // the epilogue is done with band g - 1
        {
          const int r0 = mh * 64 + 16 * (tid >> 5) + ((tid & 31) >> 2), c0 = nh * 128 + 2 * (tid & 3);
          uint8_t* d0 = sD + r0 * kOtfDumpPitch + c0 * 2;
          const float s = a.scale;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            *reinterpret_cast<uint32_t*>(d0 + 16 * j) = otf_pack2<T>(d[4 * j + 0] * s, d[4 * j + 1] * s);
            *reinterpret_cast<uint32_t*>(d0 + 8 * kOtfDumpPitch + 16 * j) = otf_pack2<T>(d[4 * j + 2] * s, d[4 * j + 3] * s);
          }
        }
       }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->dump_full);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->a_empty);  // every MMA of this warp has read its operands
    }
  } else {
    // ================= epilogue: region, accumulator dump, window blend, output =================
    const int q_local = threadIdx.x & 127;  // (row in tile) * 16 + (column in tile)
    const int half = threadIdx.x >> 7;      // 0 / 1: which half of the accumulator columns and which window rows this thread takes
    struct Geom {
      int x0, y0, b, tx, ty, l;
      float w00, w10, w01, w11;
      bool q_in, live;
      size_t q;
    };
    // window geometry of this thread's query for an item
    auto geometry = [&](int item, Geom& g) {
      const int tile = item / a.levels;
      g.l = item - tile * a.levels;
      g.tx = tile % a.tiles_x;
      g.ty = (tile / a.tiles_x) % a.tiles_y;
      g.b = tile / (a.tiles_x * a.tiles_y);
      const int qy = g.ty * 8 + (q_local >> 4), qx = g.tx * 16 + (q_local & 15);
      g.q_in = qy < a.H && qx < a.W;
      g.q = ((size_t)g.b * a.H + (g.q_in ? qy : 0)) * a.W + (g.q_in ? qx : 0);
      g.x0 = g.y0 = 0;
      g.w00 = g.w10 = g.w01 = g.w11 = 0.f;
      g.live = false;  // the window overlaps the map (otherwise all 81 outputs are zero)
      if (g.q_in) {
        const float2 c = __ldg(reinterpret_cast<const float2*>(a.coords) + g.q);
        const float sc = 1.0f / (float)(1 << g.l);
        const float x = c.x * sc, y = c.y * sc;
        const bool finite = (fabsf(x) < 1e7f) && (fabsf(y) < 1e7f);
        const float xf = finite ? floorf(x) : -1e6f, yf = finite ? floorf(y) : -1e6f;
        const float fx = finite ? x - xf : 0.f, fy = finite ? y - yf : 0.f;
        g.w00 = (1.f - fx) * (1.f - fy);  // (the dump rows already carry the scale)
        g.w10 = fx * (1.f - fy);
        g.w01 = (1.f - fx) * fy;
        g.w11 = fx * fy;
        g.x0 = (int)xf - R;
        g.y0 = (int)yf - R;
        // (selects, not a.lw[g.l]: a dynamic index into the kernel parameters makes ptxas copy them to a stack frame)
        const int Wl = g.l == 0 ? a.lw[0] : (g.l == 1 ? a.lw[1] : (g.l == 2 ? a.lw[2] : a.lw[3]));
        const int Hl = g.l == 0 ? a.lh[0] : (g.l == 1 ? a.lh[1] : (g.l == 2 ? a.lh[2] : a.lh[3]));
        g.live = g.x0 + D - 1 >= 0 && g.x0 < Wl && g.y0 + D - 1 >= 0 && g.y0 < Hl;
      }
    };
    // region of item number n: anchored at the smallest window origin of the live queries; published for the other two roles
    auto publish = [&](int n, const Geom& g) {
      int mx = g.live ? g.x0 : 0x7fffffff, my = g.live ? g.y0 : 0x7fffffff, My = g.live ? g.y0 : -0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        mx = min(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        my = min(my, __shfl_xor_sync(0xffffffffu, my, o));
        My = max(My, __shfl_xor_sync(0xffffffffu, My, o));
      }
      if (lane == 0 && warp < 4) {
        bars->red[warp][0] = mx;
        bars->red[warp][1] = my;
        bars->red[warp][2] = My;
      }
      named_barrier_sync(1, 256);
      if (threadIdx.x == 0) {
        int bx = 0x7fffffff, by = 0x7fffffff, By = -0x7fffffff;
        for (int w = 0; w < 4; ++w) {  // warps 4-7 hold the same queries
          bx = min(bx, bars->red[w][0]);
          by = min(by, bars->red[w][1]);
          By = max(By, bars->red[w][2]);
        }
        int nb = 0;
        if (bx != 0x7fffffff) {
          nb = (By + D - 1 - by + 6) / 7;  // bands of 8 rows at stride 7 that cover region rows 0 .. By + D - 1 - by
          nb = nb < 1 ? 1 : (nb > kOtfMaxBands ? kOtfMaxBands : nb);
        } else {
          bx = by = 0;
        }
        const int slot = n & 1;
        mbar_wait(&bars->reg_empty[slot], ((n >> 1) & 1) ^ 1);  // item n - 2's region has been read by both consumers
        bars->region[slot][0] = bx;
        bars->region[slot][1] = by;
        bars->region[slot][2] = nb;
        mbar_arrive(&bars->reg_full[slot]);
      }
      named_barrier_sync(1, 256);  // region[slot] readable by the epilogue threads; red[] free again
    };

    Geom cur, nxt;
    int n = 0, g = 0;
    int item = blockIdx.x;
    if (item < n_items) {
      geometry(item, cur);
      publish(0, cur);
    }
    for (; item < n_items; item += gridDim.x, ++n) {
      if (threadIdx.x == 0) OTF_TR(0);
      const int next_item = item + gridDim.x;
      if (next_item < n_items) {  // one item ahead: the producer fetches its operands during this item's blends
        geometry(next_item, nxt);
        publish(n + 1, nxt);
      }
      if (threadIdx.x == 0) OTF_TR(1);
      const int bx0 = bars->region[n & 1][0], by0 = bars->region[n & 1][1], nb = bars->region[n & 1][2];
      if (threadIdx.x == 0 && a.trace && n == 1) a.trace[blockIdx.x * 64 + 2] = (unsigned long long)nb;
      const int cxo = cur.x0 - bx0, ryo = cur.y0 - by0;  // column / row of the window's first tap inside the region
      // a window the region cannot hold: too far right of the anchor, or below the last band
      const bool outlier = cur.live && (cxo + D > kOtfRW || ryo + D - 1 > 7 * nb);
      if (cur.q_in && outlier && half == 0) a.flags[cur.q] = 1;
      const bool mine = cur.live && !outlier;
      unsigned short* orow = sOut + q_local * SP;
      if (!mine) {
        for (int c = half; c < KK; c += 2) orow[c] = 0;  // zero window (or a flagged query: its row is rewritten by the SIMT pass)
      }
      const float w00 = cur.w00, w10 = cur.w10, w01 = cur.w01, w11 = cur.w11;
      uint8_t* drow = sD + q_local * kOtfDumpPitch;
      for (int kb = 0; kb < nb; ++kb, ++g) {
        mbar_wait(&bars->dump_full, g & 1);  // band kb's dump rows are written
        if (threadIdx.x == 0) OTF_TR(8 + kb * 6 + 3);
        // ---- gather: the window rows j (of this thread's parity) whose tap pair (region rows ryo + j, ryo + j + 1) lies in
        // this band.  4-byte loads of the aligned words that cover the 2r+2 taps, realigned by a funnel shift ----
        if (mine) {
          const uint32_t* dr = reinterpret_cast<const uint32_t*>(drow);
          const uint32_t sh = (uint32_t)(cxo & 1) * 16u;
#pragma unroll 1
          for (int j = half; j < K; j += 2) {
            const int rr = ryo + j - 7 * kb;  // region row of the upper tap, relative to the band
            if (rr < 0 || rr > 6) continue;
            const uint32_t* p0 = dr + ((rr * kOtfRW + cxo) >> 1);
            uint32_t wu[D / 2 + 1], wd[D / 2 + 1];
#pragma unroll
            for (int i = 0; i <= D / 2; ++i) {
              wu[i] = p0[i];
              wd[i] = p0[i + kOtfRW / 2];
            }
            float up[D], dn[D];
#pragma unroll
            for (int i = 0; i < D / 2; ++i) {
              const uint32_t vu = __funnelshift_r(wu[i], wu[i + 1], sh), vd = __funnelshift_r(wd[i], wd[i + 1], sh);
              up[2 * i] = otf_bits_to_f32<T>((unsigned short)(vu & 0xFFFFu));
              up[2 * i + 1] = otf_bits_to_f32<T>((unsigned short)(vu >> 16));
              dn[2 * i] = otf_bits_to_f32<T>((unsigned short)(vd & 0xFFFFu));
              dn[2 * i + 1] = otf_bits_to_f32<T>((unsigned short)(vd >> 16));
            }
#pragma unroll
            for (int i = 0; i < K; ++i)
              orow[i * K + j] = otf_f32_to_bits<T>(w00 * up[i] + w10 * up[i + 1] + w01 * dn[i] + w11 * dn[i + 1]);
          }
        }
        if (threadIdx.x == 0) OTF_TR(8 + kb * 6 + 4);
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->dump_empty);  // this warp's queries are done with their dump rows: the next band may land
      }
      // ---- the level's 81 outputs of the 128 queries: coalesced 2-byte runs (81 consecutive channels per query), four rows
      // per round so that a warp has 12 loads, then 12 stores in flight ----
      named_barrier_sync(1, 256);
      {
        unsigned short* outp = reinterpret_cast<unsigned short*>(a.out);
        for (int r0 = warp; r0 < 128; r0 += 32) {
          unsigned short v[4][3];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const unsigned short* src = sOut + (r0 + 8 * u) * SP;
            v[u][0] = src[lane];
            v[u][1] = src[lane + 32];
            v[u][2] = lane + 64 < KK ? src[lane + 64] : (unsigned short)0;
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int rq = r0 + 8 * u;
            const int yy = cur.ty * 8 + (rq >> 4), xx = cur.tx * 16 + (rq & 15);
            if (yy >= a.H || xx >= a.W) continue;
            unsigned short* dst = outp + (((size_t)cur.b * a.H + yy) * a.W + xx) * a.out_stride + cur.l * KK;
            dst[lane] = v[u][0];
            dst[lane + 32] = v[u][1];
            if (lane + 64 < KK) dst[lane + 64] = v[u][2];
          }
        }
      }
      named_barrier_sync(1, 256);  // sOut (and the dump rows) are free for the next item
      if (threadIdx.x == 0) OTF_TR(3);
      // pad columns of the pixel-major rows (out_stride > levels * 81): zero
      if (cur.q_in && cur.l == 0 && half == 0) {
        unsigned short* dst = reinterpret_cast<unsigned short*>(a.out) + cur.q * a.out_stride;
        for (int c = a.levels * KK; c < a.out_stride; ++c) dst[c] = 0;
      }
      cur = nxt;
    }
  }
#undef OTF_TR
}

// ------------------------------------------------------------------------------------------------
int corr_onthefly_simt_flagged(const void* fmap1, void* const* pyr, const float* coords, void* out, const unsigned char* flags, int B, int H,
                               int W, int C, int levels, int radius, pfb_dtype dtype, int out_stride, cudaStream_t s, float scale);  // corr.cu

bool corr_onthefly_umma_supported(int B, int H, int W, int C, int levels, int radius, pfb_dtype dt, int out_stride) {
  if (dt != PFB_F16 && dt != PFB_BF16) return false;
  if (radius != 4 || levels < 1 || levels > 4) return false;
  if (C % 64 != 0 || C > 256) return false;
  if (out_stride < levels * 81) return false;
  return B > 0 && H > 0 && W > 0;
}

int corr_onthefly_umma(const void* fmap1, void* const* pyr, const float* coords, void* out, unsigned char* flags, int B, int H, int W, int C,
                       int levels, pfb_dtype dt, int out_stride, cudaStream_t s, float scale) {
  OtfArgs a{};
  a.coords = coords; a.out = out; a.flags = flags;
  a.B = B; a.H = H; a.W = W; a.kchunks = C / 64; a.levels = levels; a.out_stride = out_stride;
  a.scale = scale != 0.f ? scale : 1.0f / sqrtf((float)C);  // fmap rows wider than the features (zero channels) pass the real C's
  a.tiles_x = ceil_div(W, 16); a.tiles_y = ceil_div(H, 8); a.n_tiles = a.tiles_x * a.tiles_y * B;
  CUtensorMap tmA, tmB[4];
  {
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)W * C * 2, (uint64_t)H * W * C * 2};
    uint32_t box[4] = {64, 16, 8, 1};
    int rc = make_tensor_map(&tmA, fmap1, dt, 4, dims, str, box);
    if (rc) return rc;
  }
  for (int l = 0; l < 4; ++l) {
    const int ll = l < levels ? l : 0;
    a.lh[l] = H >> ll; a.lw[l] = W >> ll;
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)a.lw[l], (uint64_t)a.lh[l], (uint64_t)B};
    uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)a.lw[l] * C * 2, (uint64_t)a.lh[l] * a.lw[l] * C * 2};
    uint32_t box[4] = {64, (uint32_t)kOtfRW, 4, 1};  // one band half
    int rc = make_tensor_map(&tmB[l], pyr[ll], dt, 4, dims, str, box);
    if (rc) return rc;
  }
  PFB_CUDA(cudaMemsetAsync(flags, 0, (size_t)B * H * W, s));
  // shared memory: query tile + operand ring + accumulator dump + output staging; the ring takes what is left (4 stages at C = 256)
  const size_t fixed = (size_t)a.kchunks * kOtfTileBytes + 128 * kOtfDumpPitch + ((128 * 82 * 2 + 15) & ~15) + sizeof(OtfBars) + 1024;
  int stages = (int)((227 * 1024 - fixed) / kOtfTileBytes);
  if (stages > kOtfMaxStages) stages = kOtfMaxStages;
  if (stages < 2) {
    set_error("corr_lookup_onthefly_tc: no room for the operand ring (C=%d)", C);
    return PFB_ERR_UNSUPPORTED;
  }
  a.b_stages = stages;
  const size_t smem = fixed + (size_t)stages * kOtfTileBytes;
  int grid = sm_count();
  if (grid > a.n_tiles) grid = a.n_tiles;
  // PFB_OTF_TRACE=<file>: per-CTA phase timeline of the second work item (clock64 at the role hand-overs), appended as JSON lines
  static const char* trace_path = getenv("PFB_OTF_TRACE");
  if (trace_path) {
    PFB_CUDA(cudaMalloc(&a.trace, (size_t)grid * 64 * sizeof(unsigned long long)));
    PFB_CUDA(cudaMemsetAsync(a.trace, 0, (size_t)grid * 64 * sizeof(unsigned long long), s));
  }
  {
    ProfScope prof(KC_ONTHEFLY, s);
    if (dt == PFB_F16) {
      PFB_CUDA(cudaFuncSetAttribute(corr_onthefly_umma_kernel<__half, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      corr_onthefly_umma_kernel<__half, 4><<<grid, kOtfThreads, smem, s>>>(tmA, tmB[0], tmB[1], tmB[2], tmB[3], a);
    } else {
      PFB_CUDA(cudaFuncSetAttribute(corr_onthefly_umma_kernel<__nv_bfloat16, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      corr_onthefly_umma_kernel<__nv_bfloat16, 4><<<grid, kOtfThreads, smem, s>>>(tmA, tmB[0], tmB[1], tmB[2], tmB[3], a);
    }
    PFB_LAUNCH_CHECK();
  }
  if (trace_path) {
    std::vector<unsigned long long> host((size_t)grid * 64);
    PFB_CUDA(cudaStreamSynchronize(s));
    PFB_CUDA(cudaMemcpy(host.data(), a.trace, host.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    PFB_CUDA(cudaFree(a.trace));
    if (FILE* f = fopen(trace_path, "a")) {
      fprintf(f, "{\"grid\": %d, \"kchunks\": %d, \"H\": %d, \"W\": %d, \"stamps\": [", grid, a.kchunks, H, W);
      for (size_t i = 0; i < host.size(); ++i) fprintf(f, "%s%llu", i ? "," : "", host[i]);
      fprintf(f, "]}\n");
      fclose(f);
    }
  }
  // queries whose windows did not fit their tile's region: the SIMT kernel, one warp per flagged query
  return corr_onthefly_simt_flagged(fmap1, pyr, coords, out, flags, B, H, W, C, levels, 4, dt, out_stride, s, a.scale);
}

}  // namespace pfb

extern "C" PFB_API size_t pfb_corr_lookup_onthefly_tc_workspace_bytes(int B, int H, int W) {
  return B > 0 && H > 0 && W > 0 ? (size_t)B * H * W : 0;
}

extern "C" PFB_API int pfb_corr_lookup_onthefly_tc(const void* fmap1, void* const* fmap2_pyramid, const float* coords, void* out,
                                                   void* workspace, int B, int H, int W, int C, int levels, int radius, pfb_dtype dtype,
                                                   int out_stride, pfb_stream stream) {
  return pfb_corr_lookup_onthefly_tc_ex(fmap1, fmap2_pyramid, coords, out, workspace, B, H, W, C, levels, radius, 0.f, dtype, out_stride,
                                        stream);
}

extern "C" PFB_API int pfb_corr_lookup_onthefly_tc_ex(const void* fmap1, void* const* fmap2_pyramid, const float* coords, void* out,
                                                      void* workspace, int B, int H, int W, int C, int levels, int radius, float scale,
                                                      pfb_dtype dtype, int out_stride, pfb_stream stream) {
  using namespace pfb;
  PFB_CHECK_ARG(fmap1 && fmap2_pyramid && coords && out && workspace, "corr_lookup_onthefly_tc: null pointer");
  PFB_CHECK_ARG(scale >= 0.f, "corr_lookup_onthefly_tc: scale=%g", (double)scale);
  for (int l = 0; l < levels && l < 4; ++l) PFB_CHECK_ARG(fmap2_pyramid[l], "corr_lookup_onthefly_tc: fmap2 level %d is null", l);
  PFB_CHECK_ARG((H >> (levels - 1)) >= 1 && (W >> (levels - 1)) >= 1, "corr_lookup_onthefly_tc: grid too small for %d levels", levels);
  if (!corr_onthefly_umma_supported(B, H, W, C, levels, radius, dtype, out_stride)) {
    set_error("corr_lookup_onthefly_tc: needs f16/bf16, radius 4, 1-4 levels, C a multiple of 64 <= 256 (C=%d r=%d L=%d dtype=%d)", C, radius, levels, (int)dtype);
    return PFB_ERR_UNSUPPORTED;
  }
  return corr_onthefly_umma(fmap1, fmap2_pyramid, coords, out, reinterpret_cast<unsigned char*>(workspace), B, H, W, C, levels, dtype, out_stride,
                            as_stream(stream), scale);
}
