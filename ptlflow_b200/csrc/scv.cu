// a21: SCV's sparse-pyramid lookup (ptlflow/models/scv/scv.py:248-298, utils.py:148-175); the k-NN it starts from is
// pfb_knn_topk (knn_umma.cu).
//
// pfb_sparse_prepare: once per forward: the per-query table (ty + wy, tx + wx, corr) fp32 from (val, idx) and the start coordinates
//                     (w = coords - grid, the warm start), so that the loop's displacement is entry - coords1 with no state of its own.
// pfb_sparse_lookup:  once per iteration, one warp per query: the 405 bins in shared memory, then match j's 20 corner contributions
//                     (5 levels x 4 corners, all in distinct bins) added by lanes 0..19 at step j; the same order every run.
#include <math.h>

#include "common.cuh"

namespace pfb {

constexpr int KNN_MAX_K = 32;
constexpr int SCV_LEVELS = 5, SCV_RANGE = 4, SCV_BINS = 81, SCV_PLANES = SCV_LEVELS * SCV_BINS;

constexpr int SP_THREADS = 256;

__global__ void __launch_bounds__(SP_THREADS)
sparse_prepare_kernel(const float* __restrict__ val, const int* __restrict__ idx, const float* __restrict__ coords, float* __restrict__ table,
                      size_t P, int H, int W, int k) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= P * k) return;
  const size_t q = e / k;
  const int n = (int)(q % ((size_t)H * W));
  const float wx = coords[2 * q] - (float)(n % W), wy = coords[2 * q + 1] - (float)(n / W);
  const int t = idx[e];
  float* o = table + 3 * e;
  o[0] = (float)(t / W) + wy;
  o[1] = (float)(t % W) + wx;
  o[2] = val[e];
}

constexpr int SL_WARPS = 8;

template <typename T>
__global__ void __launch_bounds__(SL_WARPS * 32)
sparse_lookup_kernel(const float* __restrict__ table, const float* __restrict__ coords, T* __restrict__ out, size_t P, int k,
                     int out_stride) {
  __shared__ float bins[SL_WARPS][SCV_PLANES];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t q = (size_t)blockIdx.x * SL_WARPS + warp;
  if (q >= P) return;  // whole warps leave together
  float* bw = bins[warp];
  for (int i = lane; i < SCV_PLANES; i += 32) bw[i] = 0.f;
  const float cx = coords[2 * q], cy = coords[2 * q + 1];
  float dy = 0.f, dx = 0.f, cv = 0.f;
  if (lane < k) {
    const float* e = table + (q * k + lane) * 3;
    dy = e[0] - cy; dx = e[1] - cx; cv = e[2];
  }
  // lane l < 20: level l >> 2, corner l & 3 (0: (yf, xf), 1: (yc, xf), 2: (yf, xc), 3: (yc, xc), utils.py:159-170)
  const int lvl = lane >> 2, corner = lane & 3;
  const float s = 1.f / (float)(1 << (lvl < SCV_LEVELS ? lvl : 0));
  __syncwarp();
  for (int j = 0; j < k; ++j) {
    const float my = __shfl_sync(0xffffffffu, dy, j), mx = __shfl_sync(0xffffffffu, dx, j), mv = __shfl_sync(0xffffffffu, cv, j);
    if (lane < 4 * SCV_LEVELS) {
      const float y = my * s, x = mx * s;
      const float yf = floorf(y), xf = floorf(x);
      const float yc = yf + 1.f, xc = xf + 1.f;
      const float py = (corner & 1) ? yc : yf, px = (corner & 2) ? xc : xf;
      const float wy = (corner & 1) ? (y - yf) : (yc - y), wx = (corner & 2) ? (x - xf) : (xc - x);
      if (fabsf(py) <= (float)SCV_RANGE && fabsf(px) <= (float)SCV_RANGE)
        bw[lvl * SCV_BINS + ((int)py + SCV_RANGE) * 9 + ((int)px + SCV_RANGE)] += (wy * wx) * mv;
    }
    __syncwarp();
  }
  T* o = out + q * out_stride;
  for (int i = lane; i < out_stride; i += 32) o[i] = from_f32<T>(i < SCV_PLANES ? bw[i] : 0.f);
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_sparse_prepare(const float* val, const int* idx, const float* coords, float* table, int B, int H, int W, int k,
                                          pfb_stream stream) {
  PFB_CHECK_ARG(val && idx && coords && table, "sparse_prepare: null pointer");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && k >= 1 && k <= KNN_MAX_K && k <= H * W, "sparse_prepare: bad shape B=%d H=%d W=%d k=%d", B, H,
                W, k);
  const size_t P = (size_t)B * H * W;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  sparse_prepare_kernel<<<(unsigned)ceil_div_sz(P * k, SP_THREADS), SP_THREADS, 0, s>>>(val, idx, coords, table, P, H, W, k);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_sparse_lookup(const float* table, const float* coords, void* out, int B, int H, int W, int k, pfb_dtype dtype,
                                         int out_stride, pfb_stream stream) {
  PFB_CHECK_ARG(table && coords && out, "sparse_lookup: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "sparse_lookup: bad dtype %d", (int)dtype);
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && k >= 1 && k <= KNN_MAX_K && k <= H * W, "sparse_lookup: bad shape B=%d H=%d W=%d k=%d", B, H,
                W, k);
  PFB_CHECK_ARG(out_stride >= SCV_PLANES, "sparse_lookup: pixel stride %d < %d planes", out_stride, SCV_PLANES);
  const size_t P = (size_t)B * H * W;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_LOOKUP, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    sparse_lookup_kernel<T><<<(unsigned)ceil_div_sz(P, SL_WARPS), SL_WARPS * 32, 0, s>>>(table, coords, reinterpret_cast<T*>(out), P, k,
                                                                                           out_stride);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
