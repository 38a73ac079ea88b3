// a20: CSFlow's cross-strip correlation (ptlflow/models/csflow/csflow.py:227-278) as a second channel of the correlation pyramid
// (csflow.py:445-493), and the initial flow regressed from the strips (csflow.py:176-193).
//
// The strip channel of query q is separable: S[q, y2, x2] = sw[q, x2] + sh[q, y2].  A 2x2 average of a separable map is separable
// again, so level l of the pooled strip channel is A_l[x] + B_l[y] with A_l, B_l the pairwise means of the 1D arrays one level up
// (floor sizes, as avg_pool2d).  The strip channel is therefore kept as two fp32 tables per query, [sum_l W>>l] and [sum_l H>>l],
// and never materialised in 4D.  A bilinear tap with zero padding of such a level factors too:
//   sum_{a,b} wx_a wy_b vx_a vy_b (A[x_a] + B[y_b]) = (sum_a wx_a vx_a A[x_a]) (sum_b wy_b vy_b) + (sum_a wx_a vx_a) (sum_b wy_b vy_b B[y_b])
// (v: the corner is inside the level), so a (2r+1)^2 window costs 2 x (2r+1) two-tap sums per level.
//
// pfb_strip_means:   column / row means of the fmap2 branch (one thread per output element, fp32 sums, one rounding).
// pfb_strip_prepare: one warp per query: the fp32 tables of every level from sw / sh, and coords += (sum sh, sum sw).
// pfb_strip_lookup:  one warp per query: lane i < 2r+1 forms the two-tap sums of offset i on both axes of every level, then the
//                    warp writes the L (2r+1)^2 taps (scalar stores: the strip block starts 4 (2r+1)^2 elements into the row).
#include "common.cuh"

namespace pfb {

constexpr int SM_THREADS = 256;

template <typename T>
__global__ void __launch_bounds__(SM_THREADS)
strip_means_kernel(const T* __restrict__ gw, const T* __restrict__ gh, T* __restrict__ kw, T* __restrict__ kh, int B, int H, int W, int C) {
  const size_t nw = (size_t)B * W * C, n = nw + (size_t)B * H * C;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  float s = 0.f;
  if (t < nw) {  // kw[b, x, c] = mean over y of gw[b, y, x, c]
    const int c = (int)(t % C), x = (int)((t / C) % W), b = (int)(t / ((size_t)C * W));
    const T* p = gw + ((size_t)b * H * W + x) * C + c;
    for (int y = 0; y < H; ++y) s += to_f32(p[(size_t)y * W * C]);
    kw[t] = from_f32<T>(s / (float)H);
  } else {  // kh[b, y, c] = mean over x of gh[b, y, x, c]
    const size_t u = t - nw;
    const int c = (int)(u % C), y = (int)((u / C) % H), b = (int)(u / ((size_t)C * H));
    const T* p = gh + (((size_t)b * H + y) * W) * C + c;
    for (int x = 0; x < W; ++x) s += to_f32(p[(size_t)x * C]);
    kh[u] = from_f32<T>(s / (float)W);
  }
}

constexpr int SP_WARPS = 8;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// level 0 = the strip values in fp32; level l + 1 = pairwise means of level l (floor size).  Lanes of one warp read each other's
// global writes of the level above after __syncwarp (which orders the warp's memory accesses).
template <typename T>
__device__ __forceinline__ float strip_table(const T* __restrict__ src, float* __restrict__ tab, int n, int levels, int lane) {
  float s = 0.f;
  for (int i = lane; i < n; i += 32) {
    const float v = to_f32(src[i]);
    tab[i] = v;
    s += v;
  }
  int off = 0;
  for (int l = 1; l < levels; ++l) {
    __syncwarp();
    const int np = n >> (l - 1), nl = n >> l;
    for (int i = lane; i < nl; i += 32) tab[off + np + i] = 0.5f * (tab[off + 2 * i] + tab[off + 2 * i + 1]);
    off += np;
  }
  return s;
}

template <typename T>
__global__ void __launch_bounds__(SP_WARPS * 32)
strip_prepare_kernel(const T* __restrict__ sw, const T* __restrict__ sh, float* __restrict__ tab_w, float* __restrict__ tab_h,
                     float* __restrict__ coords, size_t P, int H, int W, int levels, int sum_w, int sum_h) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t q = (size_t)blockIdx.x * SP_WARPS + warp;
  if (q >= P) return;
  const float sx = warp_sum(strip_table(sw + q * W, tab_w + q * sum_w, W, levels, lane));
  const float sy = warp_sum(strip_table(sh + q * H, tab_h + q * sum_h, H, levels, lane));
  // corr_init = (sum over y2 of sh, sum over x2 of sw): the softmax weights of csflow.py:177-182 run over a singleton axis (all 1)
  if (coords && lane == 0) {
    coords[2 * q] += sy;
    coords[2 * q + 1] += sx;
  }
}

constexpr int SL_WARPS = 8;

// lane i < K of a warp: the two-tap sums of window offset i - r along one axis of one level: s = sum_a w_a v_a t[x_a], m = sum_a w_a v_a
__device__ __forceinline__ void strip_taps(const float* __restrict__ t, int n, float c, int r, int i, float& s, float& m) {
  const float f = floorf(c);
  s = m = 0.f;
  // a window that cannot reach the level (this also keeps huge coordinates away from the int conversion; NaN fails both tests)
  if (!(f >= -(float)(r + 1) && f <= (float)(n + r))) return;
  const float a = c - f;
  const int x0 = (int)f + i - r;
  if (x0 >= 0 && x0 < n) { s += (1.f - a) * t[x0]; m += 1.f - a; }
  if (x0 + 1 >= 0 && x0 + 1 < n) { s += a * t[x0 + 1]; m += a; }
}

template <typename T>
__global__ void __launch_bounds__(SL_WARPS * 32)
strip_lookup_kernel(const float* __restrict__ tab_w, const float* __restrict__ tab_h, const float* __restrict__ coords, T* __restrict__ out,
                    size_t P, int H, int W, int levels, int r, int sum_w, int sum_h, int out_stride, int out_offset) {
  // per warp and level: sx (sum w v A), mx (sum w v) along x, sy, my along y, one entry per window offset
  __shared__ float sm[SL_WARPS][PFB_MAX_LEVELS][4][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t q = (size_t)blockIdx.x * SL_WARPS + warp;
  if (q >= P) return;
  const int K = 2 * r + 1;
  const float cx = coords[2 * q], cy = coords[2 * q + 1];
  if (lane < K) {
    int ow = 0, oh = 0;
    for (int l = 0; l < levels; ++l) {
      const int wl = W >> l, hl = H >> l;
      const float inv = 1.f / (float)(1 << l);  // exact: coords / 2^l (corr.py's centroid_lvl)
      float s, m;
      strip_taps(tab_w + q * sum_w + ow, wl, cx * inv, r, lane, s, m);
      sm[warp][l][0][lane] = s;
      sm[warp][l][1][lane] = m;
      strip_taps(tab_h + q * sum_h + oh, hl, cy * inv, r, lane, s, m);
      sm[warp][l][2][lane] = s;
      sm[warp][l][3][lane] = m;
      ow += wl;
      oh += hl;
    }
  }
  __syncwarp();
  T* dst = out + q * out_stride + out_offset;
  const int KK = K * K, n = levels * KK;
  for (int c = lane; c < n; c += 32) {
    const int l = c / KK, rem = c - l * KK, i = rem / K, j = rem - i * K;  // channel i K + j samples (x + i - r, y + j - r)
    const float (*s)[32] = sm[warp][l];
    dst[c] = from_f32<T>(s[0][i] * s[3][j] + s[1][i] * s[2][j]);
  }
}

static int table_width(int n, int levels) {
  int s = 0;
  for (int l = 0; l < levels; ++l) s += n >> l;
  return s;
}

static int check_strip_grid(int B, int H, int W, int levels, const char* name) {
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0, "%s: bad grid %dx%dx%d", name, B, H, W);
  PFB_CHECK_ARG(levels >= 1 && levels <= PFB_MAX_LEVELS && (H >> (levels - 1)) >= 1 && (W >> (levels - 1)) >= 1,
                "%s: %dx%d grid too small for %d levels", name, H, W, levels);
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_strip_table_width(int n, int levels) {
  if (n < 1 || levels < 1 || levels > PFB_MAX_LEVELS || (n >> (levels - 1)) < 1) return 0;
  return table_width(n, levels);
}

extern "C" PFB_API int pfb_strip_means(const void* gw, const void* gh, void* kw, void* kh, int B, int H, int W, int C, pfb_dtype dtype,
                                       pfb_stream stream) {
  PFB_CHECK_ARG(gw && gh && kw && kh, "strip_means: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "strip_means: bad dtype %d", (int)dtype);
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0, "strip_means: bad shape B=%d H=%d W=%d C=%d", B, H, W, C);
  const size_t n = (size_t)B * (W + H) * C;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    strip_means_kernel<T><<<(unsigned)ceil_div_sz(n, SM_THREADS), SM_THREADS, 0, s>>>(
        reinterpret_cast<const T*>(gw), reinterpret_cast<const T*>(gh), reinterpret_cast<T*>(kw), reinterpret_cast<T*>(kh), B, H, W, C);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_strip_prepare(const void* sw, const void* sh, float* tab_w, float* tab_h, float* coords, int B, int H, int W,
                                         int levels, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(sw && sh && tab_w && tab_h, "strip_prepare: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "strip_prepare: bad dtype %d", (int)dtype);
  PFB_TRY(check_strip_grid(B, H, W, levels, "strip_prepare"));
  const size_t P = (size_t)B * H * W;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    strip_prepare_kernel<T><<<(unsigned)ceil_div_sz(P, SP_WARPS), SP_WARPS * 32, 0, s>>>(
        reinterpret_cast<const T*>(sw), reinterpret_cast<const T*>(sh), tab_w, tab_h, coords, P, H, W, levels, table_width(W, levels),
        table_width(H, levels));
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_strip_lookup(const float* tab_w, const float* tab_h, const float* coords, void* out, int B, int H, int W,
                                        int levels, int radius, pfb_dtype dtype, int out_stride, int out_offset, pfb_stream stream) {
  PFB_CHECK_ARG(tab_w && tab_h && coords && out, "strip_lookup: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "strip_lookup: bad dtype %d", (int)dtype);
  PFB_TRY(check_strip_grid(B, H, W, levels, "strip_lookup"));
  PFB_CHECK_ARG(radius >= 0 && radius <= 15, "strip_lookup: radius=%d (0..15)", radius);
  const int planes = levels * (2 * radius + 1) * (2 * radius + 1);
  PFB_CHECK_ARG(out_offset >= 0 && out_stride >= out_offset + planes, "strip_lookup: %d planes at offset %d exceed the pixel stride %d",
                planes, out_offset, out_stride);
  const size_t P = (size_t)B * H * W;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_LOOKUP, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    strip_lookup_kernel<T><<<(unsigned)ceil_div_sz(P, SL_WARPS), SL_WARPS * 32, 0, s>>>(
        tab_w, tab_h, coords, reinterpret_cast<T*>(out), P, H, W, levels, radius, table_width(W, levels), table_width(H, levels),
        out_stride, out_offset);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
