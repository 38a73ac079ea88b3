// MS-RAFT+ resampling kernels (ptlflow/models/ms_raft_plus/): the 2x bilinear upsample of the encoders' up path written straight
// into the up layer's concatenated input, the convex 2x upsample of the scale loop (of the flow, or of the absolute coordinates at
// a scale handover) and the align_corners=True resample that gives flow_small.
#include <algorithm>

#include "common.cuh"

namespace pfb {

template <typename T>
struct Vec8 {  // 8 channels, one 16-byte access for 2-byte types
  static __device__ __forceinline__ void load(const T* p, float (&f)[8]) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = to_f32(h[i]);
  }
  static __device__ __forceinline__ void store(T* p, const float (&f)[8]) {
    uint4 u;
    T* h = reinterpret_cast<T*>(&u);
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = from_f32<T>(f[i]);
    *reinterpret_cast<uint4*>(p) = u;
  }
};
template <>
struct Vec8<float> {
  static __device__ __forceinline__ void load(const float* p, float (&f)[8]) {
    float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  static __device__ __forceinline__ void store(float* p, const float (&f)[8]) {
    reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
};

// source index of F.interpolate(bilinear, align_corners=False) for an exact 2x: (o + 0.5) / 2 - 0.5, clamped at 0
__device__ __forceinline__ void src_index_2x(int o, int n, int& i0, int& i1, float& l1) {
  float s = 0.5f * ((float)o + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  i0 = (int)s;
  i1 = i0 + (i0 < n - 1 ? 1 : 0);
  l1 = s - (float)i0;
}

// out[b, y, x, 0:Cs] = bilinear2x(src)[b, y, x, :];  out[b, y, x, Cs:Cs+Ck] = skip[b, y, x, :].  One thread per (output pixel, octet).
template <typename T>
__global__ void upsample2x_concat_kernel(const T* __restrict__ src, int Cs, const T* __restrict__ skip, int Ck, T* __restrict__ out,
                                         int B, int H, int W) {
  const int OH = 2 * H, OW = 2 * W, Co = Cs + Ck, oct = Co / 8;
  const size_t total = (size_t)B * OH * OW * oct;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int o8 = (int)(idx % oct);
    const size_t p = idx / oct;  // output pixel
    const int ox = (int)(p % OW);
    const size_t t = p / OW;
    const int oy = (int)(t % OH), b = (int)(t / OH);
    const int c = 8 * o8;
    float v[8];
    if (c < Cs) {
      int y0, y1, x0, x1;
      float ly, lx;
      src_index_2x(oy, H, y0, y1, ly);
      src_index_2x(ox, W, x0, x1, lx);
      const float hy = 1.f - ly, hx = 1.f - lx;
      const T* base = src + (size_t)b * H * W * Cs + c;
      float a[8], bb[8], cc[8], d[8];
      Vec8<T>::load(base + ((size_t)y0 * W + x0) * Cs, a);
      Vec8<T>::load(base + ((size_t)y0 * W + x1) * Cs, bb);
      Vec8<T>::load(base + ((size_t)y1 * W + x0) * Cs, cc);
      Vec8<T>::load(base + ((size_t)y1 * W + x1) * Cs, d);
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = hy * (hx * a[k] + lx * bb[k]) + ly * (hx * cc[k] + lx * d[k]);
    } else {
      Vec8<T>::load(skip + p * Ck + (c - Cs), v);
    }
    Vec8<T>::store(out + p * Co + c, v);
  }
}

// Convex 2x (ms_raft_plus.py:138-149 with scale = 2): one thread per (coarse pixel, sy, sx); mask channel = tap*4 + sy*2 + sx.
// The 3x3 neighbourhood is unfolded with zero padding.  mode 0: the flow coords - grid, into the window of the un-padded NCHW
// output; mode 1: the absolute coordinates, into the next scale's pixel-major [B,2H,2W,2] coordinates; mode 2 (pfb_convex_handover2x): the flow, plus the
// fine grid, into the next scale's pixel-major coordinates (CCMR's handover, ccmr.py:195-202).
template <typename T>
__global__ void __launch_bounds__(256) convex_upsample2x_kernel(const float* __restrict__ coords, const T* __restrict__ mask,
                                                                float* __restrict__ out, int mode, int B, int H, int W, int OH, int OW,
                                                                int pad_top, int pad_left) {
  const size_t P = (size_t)B * H * W;
  const size_t tid = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const size_t p = tid >> 2;
  if (p >= P) return;
  const int sub = (int)(tid & 3), sy = sub >> 1, sx = sub & 1;
  const int x = (int)(p % W), y = (int)((p / W) % H), b = (int)(p / ((size_t)W * H));
  const T* m = mask + p * 36 + sub;
  float v[9], mx = -INFINITY;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    v[t] = to_f32(m[t * 4]);
    mx = fmaxf(mx, v[t]);
  }
  float sum = 0.f, ax = 0.f, ay = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int ny = y + t / 3 - 1, nx = x + t % 3 - 1;
    const float e = expf(v[t] - mx);
    sum += e;
    if (ny >= 0 && ny < H && nx >= 0 && nx < W) {
      const float* c = coords + 2 * ((size_t)(b * H + ny) * W + nx);
      const float gx = mode == 1 ? 0.f : (float)nx, gy = mode == 1 ? 0.f : (float)ny;
      ax = fmaf(e, 2.f * (c[0] - gx), ax);
      ay = fmaf(e, 2.f * (c[1] - gy), ay);
    }
  }
  const float inv = 1.f / sum;
  const int oy = 2 * y + sy, ox = 2 * x + sx;
  if (mode) {
    float* o = out + 2 * ((size_t)(b * 2 * H + oy) * (2 * W) + ox);
    o[0] = ax * inv;
    o[1] = ay * inv;
    if (mode == 2) {
      o[0] += (float)ox;
      o[1] += (float)oy;
    }
    return;
  }
  const int wy = oy - pad_top, wx = ox - pad_left;
  if (wy >= 0 && wy < OH && wx >= 0 && wx < OW) {
    out[((size_t)(b * 2 + 0) * OH + wy) * OW + wx] = ax * inv;
    out[((size_t)(b * 2 + 1) * OH + wy) * OW + wx] = ay * inv;
  }
}

// downflow (ms_raft_plus.py:22-35): bilinear, align_corners=True, [B,2,H,W] -> [B,2,OH,OW], u scaled by OW/W and v by OH/H
__global__ void downflow_kernel(const float* __restrict__ flow, float* __restrict__ out, int B, int H, int W, int OH, int OW, float su,
                                float sv) {
  const size_t total = (size_t)B * OH * OW;
  const float rh = OH > 1 ? (float)(H - 1) / (float)(OH - 1) : 0.f;
  const float rw = OW > 1 ? (float)(W - 1) / (float)(OW - 1) : 0.f;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % OW);
    const size_t t = idx / OW;
    const int oy = (int)(t % OH), b = (int)(t / OH);
    const float fy = rh * (float)oy, fx = rw * (float)ox;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float* f = flow + (size_t)(b * 2 + c) * H * W;
      const float v = hy * (hx * f[(size_t)y0 * W + x0] + lx * f[(size_t)y0 * W + x1]) +
                      ly * (hx * f[(size_t)y1 * W + x0] + lx * f[(size_t)y1 * W + x1]);
      out[((size_t)(b * 2 + c) * OH + oy) * OW + ox] = v * (c == 0 ? su : sv);
    }
  }
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_upsample2x_concat(const void* src, int src_channels, const void* skip, int skip_channels, void* out, int B, int H,
                                             int W, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(src && out && (skip || skip_channels == 0), "upsample2x_concat: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0, "upsample2x_concat: bad shape");
  PFB_CHECK_ARG(src_channels > 0 && src_channels % 8 == 0 && skip_channels >= 0 && skip_channels % 8 == 0,
                "upsample2x_concat: channel counts %d, %d must be multiples of 8", src_channels, skip_channels);
  PFB_CHECK_ARG(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(skip) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
                "upsample2x_concat: pointers must be 16-byte aligned");
  cudaStream_t s = as_stream(stream);
  const size_t total = (size_t)B * 4 * H * W * ((src_channels + skip_channels) / 8);
  const unsigned blocks = (unsigned)std::min<size_t>(ceil_div_sz(total, 256), (size_t)sm_count() * 32);
  ProfScope prof(KC_ENC_AFFINE, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    upsample2x_concat_kernel<T><<<blocks, 256, 0, s>>>((const T*)src, src_channels, (const T*)skip, skip_channels, (T*)out, B, H, W);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_convex_upsample2x(const float* coords, const void* mask, float* out, int mode, int B, int H, int W, int out_h,
                                             int out_w, int pad_top, int pad_left, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(coords && mask && out, "convex_upsample2x: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0 && (mode == 0 || mode == 1), "convex_upsample2x: bad arguments (mode=%d)", mode);
  if (mode == 0)
    PFB_CHECK_ARG(out_h > 0 && out_w > 0 && pad_top >= 0 && pad_left >= 0 && out_h + pad_top <= 2 * H && out_w + pad_left <= 2 * W,
                  "convex_upsample2x: output window %dx%d+(%d,%d) outside %dx%d", out_h, out_w, pad_top, pad_left, 2 * H, 2 * W);
  cudaStream_t s = as_stream(stream);
  const size_t threads = (size_t)B * H * W * 4;
  ProfScope prof(KC_UPSAMPLE, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    convex_upsample2x_kernel<T><<<(unsigned)ceil_div_sz(threads, 256), 256, 0, s>>>(coords, (const T*)mask, out, mode, B, H, W, out_h, out_w,
                                                                                    pad_top, pad_left);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_convex_handover2x(const float* coords, const void* mask, float* out, int B, int H, int W, pfb_dtype dtype,
                                             pfb_stream stream) {
  PFB_CHECK_ARG(coords && mask && out, "convex_handover2x: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && H > 0 && W > 0, "convex_handover2x: bad arguments");
  cudaStream_t s = as_stream(stream);
  const size_t threads = (size_t)B * H * W * 4;
  ProfScope prof(KC_UPSAMPLE, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    convex_upsample2x_kernel<T><<<(unsigned)ceil_div_sz(threads, 256), 256, 0, s>>>(coords, (const T*)mask, out, 2, B, H, W, 0, 0, 0, 0);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_downflow(const float* flow, float* out, int B, int H, int W, int out_h, int out_w, pfb_stream stream) {
  PFB_CHECK_ARG(flow && out, "downflow: null pointer");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0, "downflow: bad shape %dx%d -> %dx%d", H, W, out_h, out_w);
  cudaStream_t s = as_stream(stream);
  const size_t total = (size_t)B * out_h * out_w;
  const unsigned blocks = (unsigned)std::min<size_t>(ceil_div_sz(total, 256), (size_t)sm_count() * 16);
  // the reference multiplies by the Python float new / old, which the fp32 tensor op rounds to fp32
  const float su = (float)((double)out_w / (double)W), sv = (float)((double)out_h / (double)H);
  ProfScope prof(KC_UPSAMPLE, s);
  downflow_kernel<<<blocks, 256, 0, s>>>(flow, out, B, H, W, out_h, out_w, su, sv);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
