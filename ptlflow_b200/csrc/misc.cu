// Error plumbing, weight packing, context split, coordinate init and the two upsamplers.
#include <stdarg.h>

#include <algorithm>
#include <atomic>

#include "common.cuh"
#include "softmax_row.cuh"

namespace pfb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = 148;
  }
  return cached;
}

// [Cout][Cin][KH][KW] -> [KH*KW][Cin][Cout_pad] at column col_offset
__global__ void pack_conv_weight_kernel(const void* __restrict__ src, void* __restrict__ dst, int Cout, int Cin,
                                        int KH, int KW, int Cout_pad, int col_offset, int sdt, int ddt) {
  const size_t total = (size_t)Cout * Cin * KH * KW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    // idx enumerates the destination order (tap, cin, cout) so that writes are coalesced
    int co = (int)(idx % Cout);
    size_t t = idx / Cout;
    int ci = (int)(t % Cin);
    int tap = (int)(t / Cin);
    float v = load_as_f32(src, ((size_t)co * Cin + ci) * KH * KW + tap, sdt);
    store_from_f32(dst, ((size_t)tap * Cin + ci) * Cout_pad + col_offset + co, ddt, v);
  }
}

__global__ void pack_bias_kernel(const void* __restrict__ src, float* __restrict__ dst, int n, int offset, int sdt) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[offset + i] = load_as_f32(src, i, sdt);
}

template <typename T>
__global__ void context_split_kernel(const T* __restrict__ cnet, T* __restrict__ net, T* __restrict__ inp,
                                     size_t P, int hd, int cd) {
  const int C = hd + cd;
  const size_t total = P * C;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    size_t p = idx / C;
    int c = (int)(idx - p * C);
    float v = to_f32(cnet[idx]);
    if (c < hd) net[p * hd + c] = from_f32<T>(tanhf(v));
    else inp[p * cd + (c - hd)] = from_f32<T>(fmaxf(v, 0.f));
  }
}
// same, 8 channels (16 bytes of f16 / bf16) per thread: hd, cd multiples of 8, 16-byte aligned tensors
template <typename T>
__global__ void context_split_vec8_kernel(const T* __restrict__ cnet, T* __restrict__ net, T* __restrict__ inp, size_t P, int hd, int cd) {
  static_assert(sizeof(T) == 2, "16-byte vectors of 2-byte elements");
  const int C8 = (hd + cd) / 8, h8 = hd / 8;
  const size_t total = P * C8;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t p = idx / C8;
    const int c8 = (int)(idx - p * C8);
    uint4 u = __ldg(reinterpret_cast<const uint4*>(cnet) + idx);
    T* e = reinterpret_cast<T*>(&u);
    if (c8 < h8) {
#pragma unroll
      for (int k = 0; k < 8; ++k) e[k] = from_f32<T>(tanhf(to_f32(e[k])));
      reinterpret_cast<uint4*>(net)[p * h8 + c8] = u;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) e[k] = from_f32<T>(fmaxf(to_f32(e[k]), 0.f));
      reinterpret_cast<uint4*>(inp)[p * (cd / 8) + (c8 - h8)] = u;
    }
  }
}

// Warm start: RAFT's forward_interpolate (ptlflow/utils/external/raft.py:155-185, scipy griddata(method="nearest") on
// the CPU in the reference): every pixel of the previous flow is pushed to (x + dx, y + dy); points that land strictly
// inside the image are kept; each grid pixel takes the flow of its nearest kept point.  Brute force, N^2 distance
// evaluations per sample in fp64 (the reference's points are float64 = integer grid + float32 flow, exact here too);
// ties go to the lowest source index.
__global__ void __launch_bounds__(128) forward_interpolate_kernel(const float* __restrict__ flow, float* __restrict__ out, int H, int W) {
  __shared__ double2 pts[256];
  const int N = H * W, b = blockIdx.y;
  const float* fx = flow + (size_t)b * 2 * N;
  const float* fy = fx + N;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const double qx = (double)(q % W), qy = (double)(q / W);
  double best = 1e300;
  int best_i = -1;
  for (int p0 = 0; p0 < N; p0 += 256) {
    for (int t = threadIdx.x; t < 256; t += blockDim.x) {
      const int p = p0 + t;
      double2 v = make_double2(1e150, 1e150);  // never the nearest
      if (p < N) {
        const double x1 = (double)(p % W) + (double)fx[p], y1 = (double)(p / W) + (double)fy[p];
        if (x1 > 0.0 && x1 < (double)W && y1 > 0.0 && y1 < (double)H) v = make_double2(x1, y1);
      }
      pts[t] = v;
    }
    __syncthreads();
    const int n = min(256, N - p0);
    for (int t = 0; t < n; ++t) {
      const double ddx = pts[t].x - qx, ddy = pts[t].y - qy;
      const double d = ddx * ddx + ddy * ddy;
      if (d < best) {
        best = d;
        best_i = p0 + t;
      }
    }
    __syncthreads();
  }
  if (q < N) {
    const bool ok = best_i >= 0 && best < 1e290;
    out[(size_t)b * 2 * N + q] = ok ? fx[best_i] : 0.f;
    out[(size_t)b * 2 * N + N + q] = ok ? fy[best_i] : 0.f;
  }
}

__global__ void init_coords_kernel(float* __restrict__ coords, const float* __restrict__ flow_init, int B, int H,
                                   int W) {
  const int P = B * H * W;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  int x = p % W, y = (p / W) % H, b = p / (W * H);
  float fx = 0.f, fy = 0.f;
  if (flow_init) {
    fx = flow_init[((size_t)(b * 2 + 0) * H + y) * W + x];
    fy = flow_init[((size_t)(b * 2 + 1) * H + y) * W + x];
  }
  coords[2 * (size_t)p] = (float)x + fx;
  coords[2 * (size_t)p + 1] = (float)y + fy;
}

__global__ void flow_from_coords_kernel(const float* __restrict__ coords, float* __restrict__ flow, int B, int H,
                                        int W) {
  const int P = B * H * W;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  int x = p % W, y = (p / W) % H;
  flow[2 * (size_t)p] = coords[2 * (size_t)p] - (float)x;
  flow[2 * (size_t)p + 1] = coords[2 * (size_t)p + 1] - (float)y;
}

__global__ void flow_small_kernel(const float* __restrict__ coords, float* __restrict__ flow_small, int B, int H,
                                  int W) {
  const int P = B * H * W;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  int x = p % W, y = (p / W) % H, b = p / (W * H);
  flow_small[((size_t)(b * 2 + 0) * H + y) * W + x] = coords[2 * (size_t)p] - (float)x;
  flow_small[((size_t)(b * 2 + 1) * H + y) * W + x] = coords[2 * (size_t)p + 1] - (float)y;
}

// a10, convex: one thread per (coarse pixel, sy, sx); F * F threads share a coarse pixel so the nine
// mask reads (stride F * F channels) are fully coalesced.   raft.py:112-123 (F = 8), scv.py:186-197 (F = 4)
template <typename T, int F>
__global__ void __launch_bounds__(256) convex_upsample_kernel(const float* __restrict__ coords,
                                                              const T* __restrict__ mask, float* __restrict__ out,
                                                              int B, int H, int W, int OH, int OW, int pad_top,
                                                              int pad_left) {
  constexpr int FF = F * F;
  const int P = B * H * W;
  const int p = blockIdx.x * (256 / FF) + threadIdx.x / FF;
  if (p >= P) return;
  const int sub = threadIdx.x % FF;
  const int sy = sub / F, sx = sub % F;
  const int x = p % W, y = (p / W) % H, b = p / (W * H);
  const T* m = mask + (size_t)p * 9 * FF + sub;
  float v[9], mx = -INFINITY;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    v[t] = to_f32(m[t * FF]);
    mx = fmaxf(mx, v[t]);
  }
  float sum = 0.f, ax = 0.f, ay = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int ny = y + t / 3 - 1, nx = x + t % 3 - 1;
    float e = expf(v[t] - mx);
    sum += e;
    if (ny >= 0 && ny < H && nx >= 0 && nx < W) {
      const float* c = coords + 2 * ((size_t)(b * H + ny) * W + nx);
      ax = fmaf(e, (float)F * (c[0] - (float)nx), ax);
      ay = fmaf(e, (float)F * (c[1] - (float)ny), ay);
    }
  }
  const int oy = F * y + sy - pad_top, ox = F * x + sx - pad_left;
  if (oy >= 0 && oy < OH && ox >= 0 && ox < OW) {
    const float inv = 1.f / sum;
    out[((size_t)(b * 2 + 0) * OH + oy) * OW + ox] = ax * inv;
    out[((size_t)(b * 2 + 1) * OH + oy) * OW + ox] = ay * inv;
  }
}

// a12: 8 * bilinear(align_corners=True) 8x.   raft/utils.py:94-96 (torch upsample_bilinear2d semantics)
__global__ void upflow8_kernel(const float* __restrict__ coords, float* __restrict__ out, int B, int H, int W,
                               int OH, int OW, int pad_top, int pad_left) {
  const size_t total = (size_t)B * OH * OW;
  const float rh = (H > 1) ? (float)(H - 1) / (float)(8 * H - 1) : 0.f;
  const float rw = (W > 1) ? (float)(W - 1) / (float)(8 * W - 1) : 0.f;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    int ox = (int)(idx % OW);
    size_t t = idx / OW;
    int oy = (int)(t % OH);
    int b = (int)(t / OH);
    const float sy = rh * (float)(oy + pad_top), sx = rw * (float)(ox + pad_left);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      auto f = [&](int yy, int xx) {
        return coords[2 * ((size_t)(b * H + yy) * W + xx) + c] - (float)(c == 0 ? xx : yy);
      };
      float v = (1.f - ly) * ((1.f - lx) * f(y0, x0) + lx * f(y0, x1)) + ly * ((1.f - lx) * f(y1, x0) + lx * f(y1, x1));
      out[((size_t)(b * 2 + c) * OH + oy) * OW + ox] = 8.f * v;
    }
  }
}

// in-place softmax over rows of length `cols` (one block per row, fp32 math)   gma_utils.py:74
template <typename T>
__global__ void __launch_bounds__(256) softmax_rows_kernel(T* __restrict__ x, int cols) {
  __shared__ float red[8];
  T* row = x + (size_t)blockIdx.x * cols;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) m = fmaxf(m, to_f32(row[c]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
  for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) sum += expf(to_f32(row[c]) - m);
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.f / sum;
  for (int c = threadIdx.x; c < cols; c += blockDim.x) row[c] = from_f32<T>(expf(to_f32(row[c]) - m) * inv);
}

// GMA attention with the relative-position term (gma_utils.py:6-30, 62-74): one CTA per row r = (head, b, query i = x*W + y),
// logit[u*W + v] = C[r][u*W + v] (or 0 without content) + Th[r][u - x + P - 1] + Tw[r][v - y + P - 1], softmax over the row in
// fp32 (softmax_row_smem).  The row's H + W table entries are staged in shared memory behind the row.
template <typename T, bool VEC>
__global__ void __launch_bounds__(kRowThreads) attention_softmax_relpos_kernel(const T* __restrict__ logits, const float* __restrict__ th_tab,
                                                                               const float* __restrict__ tw_tab, size_t tstride,
                                                                               T* __restrict__ attn, int H, int W, int P) {
  extern __shared__ __align__(16) float srow[];  // [N] row, then th [H], tw [W]
  __shared__ float red[kRowThreads / 32];
  const int N = H * W;
  float* th = srow + N;
  float* tw = th + H;
  const size_t r = blockIdx.x;
  const int i = (int)(r % (size_t)N), x = i / W, y = i - x * W;
  const float* thr = th_tab + r * tstride + (P - 1 - x);
  const float* twr = tw_tab + r * tstride + (P - 1 - y);
  for (int u = threadIdx.x; u < H; u += kRowThreads) th[u] = thr[u];
  for (int v = threadIdx.x; v < W; v += kRowThreads) tw[v] = twr[v];
  __syncthreads();
  softmax_row_smem<T, VEC>(logits ? logits + r * N : nullptr, attn + r * N, N, W, srow, red,
                           [&](float f, int u, int v) { return f + (th[u] + tw[v]); });
}

// [B][HW][C] -> [B][C][HW_pad], zero fill for hw >= HW (32x32 smem tile transpose)
template <typename T>
__global__ void transpose_pm_kernel(const T* __restrict__ in, T* __restrict__ out, int HW, int C, int HW_pad) {
  __shared__ T tile[32][33];
  const int b = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (p < HW && c < C) ? in[((size_t)b * HW + p) * C + c] : from_f32<T>(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    if (c < C && p < HW_pad) out[((size_t)b * C + c) * HW_pad + p] = tile[threadIdx.x][i];
  }
}

int launch_flow_from_coords(const float* coords, float* flow, int B, int H, int W, cudaStream_t s) {
  const int P = B * H * W;
  ProfScope prof(KC_MISC, s);
  flow_from_coords_kernel<<<ceil_div(P, 256), 256, 0, s>>>(coords, flow, B, H, W);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_version(void) { return 102; }
extern "C" PFB_API const char* pfb_last_error(void) { return g_err; }

extern "C" PFB_API int pfb_device_arch(void) {
  int dev = 0, major = 0, minor = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  PFB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  PFB_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  return major * 10 + minor;
}

extern "C" PFB_API int pfb_stream_create(pfb_stream* out) {
  PFB_CHECK_ARG(out, "stream_create: null pointer");
  cudaStream_t s = nullptr;
  PFB_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  *out = reinterpret_cast<pfb_stream>(s);
  return PFB_OK;
}

extern "C" PFB_API int pfb_stream_destroy(pfb_stream stream) {
  PFB_CHECK_ARG(stream, "stream_destroy: null stream");
  PFB_CUDA(cudaStreamDestroy(reinterpret_cast<cudaStream_t>(stream)));
  return PFB_OK;
}

extern "C" PFB_API int pfb_pack_conv_weight(const void* src, void* dst, int Cout, int Cin, int KH, int KW, int Cout_pad,
                                    int col_offset, pfb_dtype src_dtype, pfb_dtype dst_dtype, pfb_stream stream) {
  PFB_CHECK_ARG(src && dst, "pack_conv_weight: null pointer");
  PFB_CHECK_ARG(dtype_ok(src_dtype) && dtype_ok(dst_dtype), "pack_conv_weight: bad dtype");
  PFB_CHECK_ARG(Cout > 0 && Cin > 0 && KH > 0 && KW > 0 && col_offset >= 0 && col_offset + Cout <= Cout_pad,
                "pack_conv_weight: bad shape Cout=%d Cin=%d %dx%d pad=%d off=%d", Cout, Cin, KH, KW, Cout_pad, col_offset);
  size_t total = (size_t)Cout * Cin * KH * KW;
  unsigned blocks = (unsigned)std::min<size_t>(ceil_div_sz(total, 256), 4096);
  ProfScope prof(KC_MISC, as_stream(stream));
  pack_conv_weight_kernel<<<blocks, 256, 0, as_stream(stream)>>>(src, dst, Cout, Cin, KH, KW, Cout_pad, col_offset,
                                                                 (int)src_dtype, (int)dst_dtype);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_pack_bias(const void* src, float* dst, int n, int offset, pfb_dtype src_dtype, pfb_stream stream) {
  PFB_CHECK_ARG(src && dst && n > 0 && offset >= 0 && dtype_ok(src_dtype), "pack_bias: bad arguments");
  ProfScope prof(KC_MISC, as_stream(stream));
  pack_bias_kernel<<<ceil_div(n, 256), 256, 0, as_stream(stream)>>>(src, dst, n, offset, (int)src_dtype);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_context_split(const void* cnet, void* net, void* inp, int B, int H, int W, int hidden,
                                 int context, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(cnet && net && inp, "context_split: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0 && hidden > 0 && context > 0, "context_split: bad arguments");
  size_t P = (size_t)B * H * W;
  ProfScope prof(KC_MISC, as_stream(stream));
  const bool vec = dtype != PFB_F32 && hidden % 8 == 0 && context % 8 == 0 &&
                   ((reinterpret_cast<uintptr_t>(cnet) | reinterpret_cast<uintptr_t>(net) | reinterpret_cast<uintptr_t>(inp)) & 15) == 0;
  if (vec) {
    unsigned blocks = (unsigned)std::min<size_t>(ceil_div_sz(P * (hidden + context) / 8, 256), (size_t)sm_count() * 16);
    if (dtype == PFB_F16) context_split_vec8_kernel<__half><<<blocks, 256, 0, as_stream(stream)>>>((const __half*)cnet, (__half*)net, (__half*)inp, P, hidden, context);
    else context_split_vec8_kernel<__nv_bfloat16><<<blocks, 256, 0, as_stream(stream)>>>((const __nv_bfloat16*)cnet, (__nv_bfloat16*)net, (__nv_bfloat16*)inp, P, hidden, context);
  } else {
    unsigned blocks = (unsigned)std::min<size_t>(ceil_div_sz(P * (hidden + context), 256), (size_t)sm_count() * 16);
    PFB_DISPATCH_DTYPE(dtype, T, {
      context_split_kernel<T><<<blocks, 256, 0, as_stream(stream)>>>((const T*)cnet, (T*)net, (T*)inp, P, hidden, context);
    });
  }
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_forward_interpolate(const float* flow_nchw, float* out_nchw, int B, int H, int W, pfb_stream stream) {
  PFB_CHECK_ARG(flow_nchw && out_nchw && B > 0 && H > 0 && W > 0 && B <= 65535, "forward_interpolate: bad arguments");
  ProfScope prof(KC_MISC, as_stream(stream));
  forward_interpolate_kernel<<<dim3(ceil_div(H * W, 128), B), 128, 0, as_stream(stream)>>>(flow_nchw, out_nchw, H, W);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_init_coords(float* coords, const float* flow_init_nchw, int B, int H, int W, pfb_stream stream) {
  PFB_CHECK_ARG(coords && B > 0 && H > 0 && W > 0, "init_coords: bad arguments");
  ProfScope prof(KC_MISC, as_stream(stream));
  init_coords_kernel<<<ceil_div(B * H * W, 256), 256, 0, as_stream(stream)>>>(coords, flow_init_nchw, B, H, W);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

static int write_flow_small(const float* coords, float* flow_small, int B, int H, int W, cudaStream_t s) {
  if (!flow_small) return PFB_OK;
  ProfScope prof(KC_MISC, s);
  flow_small_kernel<<<ceil_div(B * H * W, 256), 256, 0, s>>>(coords, flow_small, B, H, W);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

template <int F>
static int convex_upsample(const float* coords, const void* mask, float* out, float* flow_small, int B, int H, int W, int out_h, int out_w,
                           int pad_top, int pad_left, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(coords && mask && out, "convex_upsample: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0, "convex_upsample: bad arguments");
  PFB_CHECK_ARG(out_h > 0 && out_w > 0 && pad_top >= 0 && pad_left >= 0 && out_h + pad_top <= F * H && out_w + pad_left <= F * W,
                "convex_upsample: output window %dx%d+(%d,%d) outside %dx%d", out_h, out_w, pad_top, pad_left, F * H, F * W);
  cudaStream_t s = as_stream(stream);
  const int P = B * H * W;
  {
  ProfScope prof(KC_UPSAMPLE, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    convex_upsample_kernel<T, F><<<ceil_div(P, 256 / (F * F)), 256, 0, s>>>(coords, (const T*)mask, out, B, H, W, out_h, out_w, pad_top,
                                                                            pad_left);
  });
  }
  PFB_LAUNCH_CHECK();
  return write_flow_small(coords, flow_small, B, H, W, s);
}

extern "C" PFB_API int pfb_convex_upsample(const float* coords, const void* mask, float* out, float* flow_small, int B,
                                   int H, int W, int out_h, int out_w, int pad_top, int pad_left,
                                   pfb_dtype dtype, pfb_stream stream) {
  return convex_upsample<8>(coords, mask, out, flow_small, B, H, W, out_h, out_w, pad_top, pad_left, dtype, stream);
}

extern "C" PFB_API int pfb_convex_upsample4x(const float* coords, const void* mask, float* out, float* flow_small, int B, int H, int W,
                                             int out_h, int out_w, int pad_top, int pad_left, pfb_dtype dtype, pfb_stream stream) {
  return convex_upsample<4>(coords, mask, out, flow_small, B, H, W, out_h, out_w, pad_top, pad_left, dtype, stream);
}

extern "C" PFB_API int pfb_upflow8(const float* coords, float* out, float* flow_small, int B, int H, int W, int out_h,
                           int out_w, int pad_top, int pad_left, pfb_stream stream) {
  PFB_CHECK_ARG(coords && out && B > 0 && H > 0 && W > 0, "upflow8: bad arguments");
  PFB_CHECK_ARG(out_h > 0 && out_w > 0 && pad_top >= 0 && pad_left >= 0 && out_h + pad_top <= 8 * H && out_w + pad_left <= 8 * W,
                "upflow8: output window outside the upsampled grid");
  cudaStream_t s = as_stream(stream);
  size_t total = (size_t)B * out_h * out_w;
  unsigned blocks = (unsigned)std::min<size_t>(ceil_div_sz(total, 256), (size_t)sm_count() * 16);
  {
    ProfScope prof(KC_UPSAMPLE, s);
    upflow8_kernel<<<blocks, 256, 0, s>>>(coords, out, B, H, W, out_h, out_w, pad_top, pad_left);
  }
  PFB_LAUNCH_CHECK();
  return write_flow_small(coords, flow_small, B, H, W, s);
}

extern "C" PFB_API int pfb_softmax_rows(void* x, size_t rows, int cols, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && rows > 0 && rows < (1ull << 31) && cols > 0 && dtype_ok(dtype), "softmax_rows: bad arguments");
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, { softmax_rows_kernel<T><<<(unsigned)rows, 256, 0, s>>>((T*)x, cols); });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

template <typename T, bool VEC>
static int launch_relpos_softmax(const void* logits, const float* th, const float* tw, size_t tstride, void* attn, size_t rows, int H,
                                 int W, int P, cudaStream_t s) {
  const size_t smem = (size_t)(H * W + H + W) * sizeof(float);
  // once per (instantiation, device): rows of more than 12 288 entries need more than the default 48 KB
  static std::atomic<unsigned long long> attr_done{0};
  int dev = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  if (!(attr_done.load(std::memory_order_acquire) & (1ull << (dev & 63)))) {
    PFB_CUDA(cudaFuncSetAttribute(attention_softmax_relpos_kernel<T, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
  }
  attention_softmax_relpos_kernel<T, VEC><<<(unsigned)rows, kRowThreads, smem, s>>>((const T*)logits, th, tw, tstride, (T*)attn, H, W, P);
  return PFB_OK;
}

extern "C" PFB_API int pfb_attention_softmax_relpos(const void* logits, const float* th, const float* tw, size_t table_stride, void* attn,
                                                    size_t rows, int H, int W, int P, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(th && tw && attn && dtype_ok(dtype), "attention_softmax_relpos: null pointer or bad dtype");
  PFB_CHECK_ARG(P > 0 && H > 0 && W > 0 && H <= P && W <= P, "attention_softmax_relpos: %dx%d grid outside the %dx%d position table", H, W, P, P);
  PFB_CHECK_ARG(table_stride >= (size_t)(2 * P - 1), "attention_softmax_relpos: table_stride %zu < 2P-1 = %d", table_stride, 2 * P - 1);
  const size_t N = (size_t)H * W;
  PFB_CHECK_ARG(rows > 0 && rows < (1ull << 31) && rows % N == 0, "attention_softmax_relpos: rows=%zu is not a multiple of H*W=%zu", rows, N);
  cudaStream_t s = as_stream(stream);
  const size_t ev = 16 / dtype_size(dtype);
  const bool vec = N % ev == 0 && ((reinterpret_cast<uintptr_t>(logits) | reinterpret_cast<uintptr_t>(attn)) & 15) == 0;
  int rc = PFB_OK;
  {
    ProfScope prof(KC_MISC, s);
    PFB_DISPATCH_DTYPE(dtype, T, {
      rc = vec ? launch_relpos_softmax<T, true>(logits, th, tw, table_stride, attn, rows, H, W, P, s)
               : launch_relpos_softmax<T, false>(logits, th, tw, table_stride, attn, rows, H, W, P, s);
    });
  }
  if (rc != PFB_OK) return rc;
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_transpose_pm(const void* in, void* out, int B, int HW, int C, int HW_pad, pfb_dtype dtype,
                                        pfb_stream stream) {
  PFB_CHECK_ARG(in && out && B > 0 && B <= 65535 && HW > 0 && C > 0 && HW_pad >= HW && dtype_ok(dtype), "transpose_pm: bad arguments");
  cudaStream_t s = as_stream(stream);
  dim3 grid(ceil_div(HW_pad, 32), ceil_div(C, 32), B), block(32, 8);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, { transpose_pm_kernel<T><<<grid, block, 0, s>>>((const T*)in, (T*)out, HW, C, HW_pad); });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
