// SplatFlow (a24): forward splatting of pixel-major features by a flow, "average" mode of softsplat.py:10-60, 435-468.
// See include/ptlflow_b200.h, a24.
#include "common.cuh"

namespace pfb {

namespace {

constexpr int kSplatWarps = 8;  // source pixels per CTA of the scatter (one warp each)

// One warp per source pixel p = (b, y, x): the target (x + u, y + v) and the bilinear weights of its four floor / floor + 1 corners
// in fp32, exactly as kernel_Softsplat_updateOutput forms them, once per pixel; then per channel the fp32 product value * weight,
// widened to double and added into acc [P][C + 1] at each in-image corner.  Lane 0 adds the weight itself (the ones channel, 1 * w)
// into column C, once per corner.
template <typename T>
__global__ void __launch_bounds__(kSplatWarps * 32) splat_scatter_kernel(const T* __restrict__ src, int src_stride, const float* __restrict__ flow,
                                                                          double* __restrict__ acc, int B, int H, int W, int C) {
  const int lane = threadIdx.x & 31;
  const size_t P = (size_t)B * H * W;
  const size_t p = (size_t)blockIdx.x * kSplatWarps + (threadIdx.x >> 5);
  if (p >= P) return;
  const int x = (int)(p % W);
  const int y = (int)((p / W) % H);
  const int b = (int)(p / ((size_t)W * H));
  const size_t plane = (size_t)H * W;
  const float fx = (float)x + flow[((size_t)b * 2 + 0) * plane + (size_t)y * W + x];
  const float fy = (float)y + flow[((size_t)b * 2 + 1) * plane + (size_t)y * W + x];
  const int x0 = (int)floorf(fx), y0 = (int)floorf(fy);
  const int x1 = x0 + 1, y1 = y0 + 1;
  // northwest, northeast, southwest, southeast (softsplat.py:34-37)
  float w[4];
  w[0] = __fmul_rn(__fsub_rn((float)x1, fx), __fsub_rn((float)y1, fy));
  w[1] = __fmul_rn(__fsub_rn(fx, (float)x0), __fsub_rn((float)y1, fy));
  w[2] = __fmul_rn(__fsub_rn((float)x1, fx), __fsub_rn(fy, (float)y0));
  w[3] = __fmul_rn(__fsub_rn(fx, (float)x0), __fsub_rn(fy, (float)y0));
  const int cx[4] = {x0, x1, x0, x1}, cy[4] = {y0, y0, y1, y1};
  double* dst[4];
#pragma unroll
  for (int k = 0; k < 4; ++k)
    dst[k] = (cx[k] >= 0 && cx[k] < W && cy[k] >= 0 && cy[k] < H) ? acc + (((size_t)b * H + cy[k]) * W + cx[k]) * (C + 1) : nullptr;
  const T* s = src + p * src_stride;
  for (int c = lane; c < C; c += 32) {
    const float v = to_f32(s[c]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (dst[k]) atomicAdd(dst[k] + c, (double)__fmul_rn(v, w[k]));
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (dst[k]) atomicAdd(dst[k] + C, (double)w[k]);
  }
}

// out[p, c] = float(acc[p, c]) / n,  n = float(acc[p, C]), or 1 where that is exactly 0 (softsplat.py:327, 460-465); fp32 division,
// one rounding to the storage type.  One thread per (pixel, channel).
template <typename T>
__global__ void __launch_bounds__(256) splat_normalize_kernel(const double* __restrict__ acc, T* __restrict__ out, int out_stride, size_t P, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P * C) return;
  const size_t p = i / C;
  const int c = (int)(i - p * C);
  const double* a = acc + p * (C + 1);
  float n = (float)a[C];
  if (n == 0.f) n = 1.f;
  out[p * out_stride + c] = from_f32<T>(__fdiv_rn((float)a[c], n));
}

}  // namespace

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API size_t pfb_softsplat_workspace_bytes(int B, int H, int W, int C) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0) return 0;
  return align_up((size_t)B * H * W * (C + 1) * sizeof(double), 256);
}

extern "C" PFB_API int pfb_softsplat_average(const void* src, int src_stride, int src_offset, const float* flow, void* dst, int dst_stride,
                                             int dst_offset, void* workspace, size_t workspace_bytes, int B, int H, int W, int C,
                                             pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(src && flow && dst && workspace && dtype_ok(dtype), "softsplat_average: null pointer or bad dtype");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0, "softsplat_average: bad shape %dx%dx%dx%d", B, H, W, C);
  PFB_CHECK_ARG(src_offset >= 0 && src_stride >= src_offset + C && dst_offset >= 0 && dst_stride >= dst_offset + C,
                "softsplat_average: strides / offsets (%d+%d, %d+%d) do not hold %d channels", src_stride, src_offset, dst_stride, dst_offset, C);
  const size_t need = pfb_softsplat_workspace_bytes(B, H, W, C);
  PFB_CHECK_ARG(workspace_bytes >= need, "softsplat_average: workspace %zu bytes < required %zu", workspace_bytes, need);
  const size_t P = (size_t)B * H * W;
  cudaStream_t s = as_stream(stream);
  double* acc = reinterpret_cast<double*>(workspace);
  ProfScope prof(KC_MISC, s);
  PFB_CUDA(cudaMemsetAsync(acc, 0, P * (C + 1) * sizeof(double), s));
  PFB_DISPATCH_DTYPE(dtype, T, {
    splat_scatter_kernel<T><<<(unsigned)ceil_div_sz(P, kSplatWarps), kSplatWarps * 32, 0, s>>>((const T*)src + src_offset, src_stride, flow,
                                                                                                  acc, B, H, W, C);
    splat_normalize_kernel<T><<<(unsigned)ceil_div_sz(P * C, 256), 256, 0, s>>>(acc, (T*)dst + dst_offset, dst_stride, P, C);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
