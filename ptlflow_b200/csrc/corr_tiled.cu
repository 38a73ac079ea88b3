// a3 on the TILED correlation pyramid (f16 / bf16 storage).
//
// Layout ("T84"): level l of query q is a grid of tiles_y x tiles_x tiles, a tile = 4 rows x 8 columns = 64 bytes =
// one DRAM access granule (the dense layout of pfb_corr_volume_build costs 64 B of DRAM traffic for every 20-byte window
// row: ncu r01, 181.6 MB read per launch for 45 MB of window data).  Element (y, x) of a map lives at element offset
//     ((y >> 2) * tiles_x + (x >> 3)) * 32 + (y & 3) * 8 + (x & 7),
// tiles_x = ceil(W_l / 8), tiles_y = ceil(H_l / 4); pad rows / columns (y >= H_l, x >= W_l inside the last tiles) are never
// relied upon: the lookup masks them.  A (2r+2)^2 = 10 x 10 window then touches (1 + 9/8) x (1 + 9/4) = 6.9 tiles on average = 442 B per level
// instead of 820 B, every byte of which arrives through 16-byte loads of whole tile rows.
//
// Kernel: one warp per query.  Phase 1: the lanes fetch, for all four levels at once (independent 128-bit loads, all in
// flight before any is consumed), the 16-byte tile rows the windows touch and park them in shared memory as
// [level][window row][3 chunks x 8 columns].  Phase 2: every lane blends output channels (x-major window order of
// ptlflow/models/raft/corr.py:43-47, zero outside the map: raft/utils.py:71-75) from that staging copy in fp32 and writes
// them to a shared-memory row, which leaves as one coalesced run of 16-byte stores.
#include "common.cuh"

namespace pfb {

struct TiledLevels {
  const void* ptr[4];
  int h[4], w[4];
  int tiles_x[4];
  unsigned map_elems[4];  // elements per query map = tiles_y * tiles_x * 32
};

__host__ __device__ inline int tiled_tiles_x(int w) { return (w + 7) >> 3; }
__host__ __device__ inline int tiled_tiles_y(int h) { return (h + 3) >> 2; }

template <typename T>
__device__ __forceinline__ float half_bits_to_f32(unsigned short b);
template <>
__device__ __forceinline__ float half_bits_to_f32<__half>(unsigned short b) { return __half2float(__ushort_as_half(b)); }
template <>
__device__ __forceinline__ float half_bits_to_f32<__nv_bfloat16>(unsigned short b) { return __uint_as_float((unsigned)b << 16); }

template <typename T>
__device__ __forceinline__ unsigned short f32_to_half_bits(float v);
template <>
__device__ __forceinline__ unsigned short f32_to_half_bits<__half>(float v) { return __half_as_ushort(__float2half_rn(v)); }
template <>
__device__ __forceinline__ unsigned short f32_to_half_bits<__nv_bfloat16>(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }

constexpr int kTlWarps = 4;

// The first version of this kernel (one loop over 120 (level, row, chunk) slots and one over 324 channels, level
// geometry and blend weights fetched through shared memory with a per-lane level index) retired 1000 instructions per
// query-warp and ran at 87 % issue utilisation with DRAM at 23 % (ncu r02b): instruction-bound.  Here the levels are
// unrolled: a lane's (window row, chunk) slot and its (i, j) output positions are the same for every level and are
// decoded once; per level only the scaled coordinates, one address and the four blend weights remain, all in registers.
template <typename T, int R, int LEVELS>
__global__ void __launch_bounds__(kTlWarps * 32) corr_lookup_tiled_kernel(const TiledLevels lv, const float* __restrict__ coords,
                                                                          T* __restrict__ out, int nq, int out_stride) {
  constexpr int D = 2 * R + 2, K = 2 * R + 1, KK = K * K;
  constexpr int ROWP = 24;                 // staged window row: 3 chunks of 8 columns (48 bytes)
  constexpr int LVP = D * ROWP;            // halfs per staged level
  constexpr int PLANES = LEVELS * KK;
  constexpr int OUTP = (PLANES + 7) / 8 * 8;
  constexpr int NPOS = K == 9 ? 3 : (K + 3) / 4;  // output positions per lane and level (rounds of 8 rows x 4 columns, see phase 2)
  static_assert(D * 3 <= 32, "one (window row, chunk) slot per lane");
  static_assert(K <= 9, "phase 2 covers windows of up to 9 x 9 positions");
  __shared__ __align__(16) unsigned short stage[kTlWarps][LEVELS * LVP];
  __shared__ __align__(16) unsigned short orow[kTlWarps][OUTP];

  pdl_wait();     // coords / volume come from the previous kernels in the stream
  pdl_trigger();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = blockIdx.x * kTlWarps + warp;
  if (q >= nq) return;
  const float2 c = __ldg(reinterpret_cast<const float2*>(coords) + q);
  unsigned short* st = stage[warp];

  // ---- phase 1: lane = (window row j, chunk ck), the same slot in every level; all levels' loads in flight together ----
  const int j1 = lane / 3, ck = lane - j1 * 3;
  const bool slot = lane < D * 3;
  // Level geometry once per warp, not once per level and lane: lane (l mod 4) works out level l's window origin and
  // bilinear fractions, the others pick them up by shuffle (phase 1 was 350 of the kernel's 550 instructions when every
  // lane redid the floor / finite / weight arithmetic for all four levels).
  int gx0, gy0;
  float gfx, gfy;
  {
    const float sc = __uint_as_float((127u - (unsigned)(lane & 3)) << 23);  // 2^-(lane & 3), exact
    const float x = c.x * sc, y = c.y * sc;
    const bool finite = (fabsf(x) < 1e7f) && (fabsf(y) < 1e7f);
    const float xf = finite ? floorf(x) : -1e6f, yf = finite ? floorf(y) : -1e6f;
    gfx = finite ? x - xf : 0.f;
    gfy = finite ? y - yf : 0.f;
    gx0 = (int)xf - R;
    gy0 = (int)yf - R;
  }
  const bool slot01 = slot && ck < 2;
  uint4 v[LEVELS];
  float w00[LEVELS], w10[LEVELS], w01[LEVELS], w11[LEVELS];
  int off[LEVELS];
#pragma unroll
  for (int l = 0; l < LEVELS; ++l) {
    const int x0 = __shfl_sync(0xffffffffu, gx0, l), y0 = __shfl_sync(0xffffffffu, gy0, l);
    const float fx = __shfl_sync(0xffffffffu, gfx, l), fy = __shfl_sync(0xffffffffu, gfy, l);
    w00[l] = (1.f - fx) * (1.f - fy);
    w10[l] = fx * (1.f - fy);
    w01[l] = (1.f - fx) * fy;
    w11[l] = fx * fy;
    const int o = x0 & 7;                  // column of the window's first tap inside its tile (two's complement: floor mod)
    off[l] = o;
    const int yy = y0 + j1, tcol = (x0 >> 3) + ck;
    v[l] = make_uint4(0u, 0u, 0u, 0u);
    // the third chunk is touched only when the 2r+2 taps starting at column o run past 16
    if ((slot01 || (slot && o + D > 16)) && (unsigned)yy < (unsigned)lv.h[l] && (unsigned)tcol < (unsigned)lv.tiles_x[l]) {
      const unsigned short* base = reinterpret_cast<const unsigned short*>(lv.ptr[l]) + (size_t)q * lv.map_elems[l];
      const unsigned e = ((unsigned)(yy >> 2) * (unsigned)lv.tiles_x[l] + (unsigned)tcol) * 32u + (unsigned)(yy & 3) * 8u;
      uint4 u = __ldg(reinterpret_cast<const uint4*>(base + e));
      if (lv.w[l] & 7) {  // kernel-uniform: only maps whose width is not a multiple of 8 have pad columns (they may hold anything)
        const int nvalid = lv.w[l] - tcol * 8;
        if (nvalid < 8) {
          u.x = nvalid >= 2 ? u.x : (nvalid == 1 ? (u.x & 0xFFFFu) : 0u);
          u.y = nvalid >= 4 ? u.y : (nvalid == 3 ? (u.y & 0xFFFFu) : 0u);
          u.z = nvalid >= 6 ? u.z : (nvalid == 5 ? (u.z & 0xFFFFu) : 0u);
          u.w = nvalid >= 8 ? u.w : (nvalid == 7 ? (u.w & 0xFFFFu) : 0u);
        }
      }
      v[l] = u;
    }
  }
  if (slot) {
#pragma unroll
    for (int l = 0; l < LEVELS; ++l) *reinterpret_cast<uint4*>(st + l * LVP + lane * 8) = v[l];  // j1 * ROWP + ck * 8 == lane * 8
  }
  __syncwarp();

  // ---- phase 2: every lane blends NPOS output positions (i, j) of the window, the same in every level.  Lane -> position is
  // chosen for the staging copy's banks: j = lane & 7, i = lane >> 3 (+ 4 per round) puts the 8 rows of one instruction 12 words
  // apart and leaves 4 bank-free words between them for the <= 3 words the 4 columns span; with position = lane + 32 k, rows 0
  // and 8 of the same instruction shared banks and every one of the 48 two-byte reads took two wavefronts (ncu r02m: the kernel
  // was L1TEX-bound at 86 %).  channel = l * KK + i * K + j, i <-> x offset (x-major, corr.py:43-47) ----
  unsigned short* ow = orow[warp];
  int tap[NPOS], opos[NPOS];
  bool act[NPOS];
#pragma unroll
  for (int k = 0; k < NPOS; ++k) {
    int i, j;
    if (K == 9 && k == 2) {  // what the 8-row rounds leave of a 9 x 9 window: column i = 8 (8 rows) and row j = 8 (9 columns)
      i = lane < 8 ? 8 : lane - 8;
      j = lane < 8 ? lane : 8;
      act[k] = lane < 17;
    } else {
      i = (lane >> 3) + 4 * k;
      j = lane & 7;
      act[k] = j < K && i < K;
    }
    tap[k] = act[k] ? j * ROWP + i : 0;
    opos[k] = i * K + j;
  }
#pragma unroll
  for (int l = 0; l < LEVELS; ++l) {
    const unsigned short* sl = st + l * LVP + off[l];
#pragma unroll
    for (int k = 0; k < NPOS; ++k) {
      if (act[k]) {
        const unsigned short* w0 = sl + tap[k];
        const float r = w00[l] * half_bits_to_f32<T>(w0[0]) + w10[l] * half_bits_to_f32<T>(w0[1]) + w01[l] * half_bits_to_f32<T>(w0[ROWP]) +
                        w11[l] * half_bits_to_f32<T>(w0[ROWP + 1]);
        ow[l * KK + opos[k]] = f32_to_half_bits<T>(r);
      }
    }
  }
  if (lane < OUTP - PLANES) ow[PLANES + lane] = 0;
  __syncwarp();
  // ---- coalesced 16-byte stores of the output row (out_stride % 8 == 0; columns beyond OUTP are zero-filled) ----
  uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<unsigned short*>(out) + (size_t)q * out_stride);
  const int chunks = out_stride >> 3;
  const uint4* ow4 = reinterpret_cast<const uint4*>(ow);
  static_assert(OUTP / 8 <= 64, "two rounds of 16-byte stores cover the output row");
  if (lane < OUTP / 8) dst[lane] = ow4[lane];
  if (lane + 32 < OUTP / 8) dst[lane + 32] = ow4[lane + 32];
  for (int k = OUTP / 8 + lane; k < chunks; k += 32) dst[k] = make_uint4(0u, 0u, 0u, 0u);  // only when the caller's rows are wider
}

template <typename T>
static int launch_lookup_tiled(const TiledLevels& lv, const float* coords, void* out, int nq, int levels, int radius, int out_stride,
                               cudaStream_t s) {
  if (!(radius == 4 || (radius == 3 && levels >= 3))) {  // refused before the launch is counted
    set_error("corr_lookup_tiled: radius=%d levels=%d not instantiated (radius 4 with 1-4 levels, radius 3 with 3-4)", radius, levels);
    return PFB_ERR_UNSUPPORTED;
  }
  dim3 grid(ceil_div(nq, kTlWarps));
  ProfScope prof(KC_LOOKUP, s);
#define PFB_TL(R, L) PFB_CUDA(launch_pdl(corr_lookup_tiled_kernel<T, R, L>, grid, dim3(kTlWarps * 32), 0, s, lv, coords, (T*)out, nq, out_stride))
  if (radius == 4 && levels == 4) PFB_TL(4, 4);
  else if (radius == 4 && levels == 3) PFB_TL(4, 3);
  else if (radius == 4 && levels == 2) PFB_TL(4, 2);
  else if (radius == 4) PFB_TL(4, 1);
  else if (levels == 4) PFB_TL(3, 4);
  else PFB_TL(3, 3);
#undef PFB_TL
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API size_t pfb_corr_level_bytes_tiled(int B, int H1, int W1, int H2, int W2, int level) {
  const int h = H2 >> level, w = W2 >> level;
  if (B <= 0 || H1 <= 0 || W1 <= 0 || h < 1 || w < 1) return 0;
  return (size_t)B * H1 * W1 * (size_t)tiled_tiles_y(h) * tiled_tiles_x(w) * 64;
}

extern "C" PFB_API int pfb_corr_lookup_tiled(void* const* pyramid, const float* coords, void* out, int B, int H, int W, int H2, int W2,
                                             int levels, int radius, pfb_dtype dtype, int out_stride, pfb_stream stream) {
  return pfb_corr_lookup_tiled_ex(pyramid, nullptr, nullptr, coords, out, B, H, W, H2, W2, levels, radius, dtype, out_stride, stream);
}

extern "C" PFB_API int pfb_corr_lookup_tiled_ex(void* const* pyramid, const int* level_h, const int* level_w, const float* coords, void* out,
                                                int B, int H, int W, int H2, int W2, int levels, int radius, pfb_dtype dtype, int out_stride,
                                                pfb_stream stream) {
  PFB_CHECK_ARG(pyramid && coords && out, "corr_lookup_tiled: null pointer");
  PFB_CHECK_ARG((level_h == nullptr) == (level_w == nullptr), "corr_lookup_tiled: level_h and level_w come together");
  PFB_CHECK_ARG(dtype == PFB_F16 || dtype == PFB_BF16, "corr_lookup_tiled: the tiled pyramid is f16 / bf16 only");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && H2 > 0 && W2 > 0, "corr_lookup_tiled: bad shape");
  PFB_CHECK_ARG(levels >= 1 && levels <= 4, "corr_lookup_tiled: levels=%d out of range (1..4)", levels);
  const int planes = levels * (2 * radius + 1) * (2 * radius + 1);
  PFB_CHECK_ARG(out_stride >= planes && out_stride % 8 == 0, "corr_lookup_tiled: out_stride=%d must be a multiple of 8 and >= %d", out_stride, planes);
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15) == 0, "corr_lookup_tiled: out must be 16-byte aligned");
  TiledLevels lv{};
  for (int l = 0; l < levels; ++l) {
    PFB_CHECK_ARG(pyramid[l] && (reinterpret_cast<uintptr_t>(pyramid[l]) & 15) == 0, "corr_lookup_tiled: pyramid[%d] null or not 16-byte aligned", l);
    lv.ptr[l] = pyramid[l];
    lv.h[l] = level_h ? level_h[l] : H2 >> l;
    lv.w[l] = level_w ? level_w[l] : W2 >> l;
    PFB_CHECK_ARG(lv.h[l] >= 1 && lv.w[l] >= 1, "corr_lookup_tiled: level %d is empty", l);
    lv.tiles_x[l] = tiled_tiles_x(lv.w[l]);
    lv.map_elems[l] = (unsigned)(tiled_tiles_y(lv.h[l]) * lv.tiles_x[l] * 32);
  }
  if (dtype == PFB_F16) return launch_lookup_tiled<__half>(lv, coords, out, B * H * W, levels, radius, out_stride, as_stream(stream));
  return launch_lookup_tiled<__nv_bfloat16>(lv, coords, out, B * H * W, levels, radius, out_stride, as_stream(stream));
}
