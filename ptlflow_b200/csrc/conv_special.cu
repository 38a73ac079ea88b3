// Two small convolutions of the update block that do not fit the tensor-core tile economically, plus
// the K-major weight packing used by the wgmma path.
//   * flow-head conv2 (3x3, 256 -> 2, update.py:9) fused with the coordinate update of raft.py:174-178:
//     one warp per pixel, lanes split the input channels with 128-bit loads, shuffle reduction.
//   * motion-encoder convf1 (7x7, 2 -> 128/64, update.py:99,:81): one thread per output channel keeps its
//     98 weights in registers and slides a 16-pixel accumulator row over a shared-memory flow patch.
#include "common.cuh"

namespace pfb {

template <typename T>
__device__ __forceinline__ void unpack8f(const uint4& u, float (&f)[8]) {
  const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = to_f32(h[i]);
}

// ---------------------------------------------------------------------------------------------
// Flow head conv2: the two weight rows of every tap are staged once per block in shared memory; each warp
// then walks pixels (grid-stride), issuing the 128-bit loads of all taps before the FMAs.
template <typename T, int KH, int KW>
__global__ void __launch_bounds__(256) conv_cout2_flow_kernel(const T* __restrict__ x, int stride, int offset, int Cin,
                                                              int B, int H, int W, const T* __restrict__ wk,
                                                              int Cout_pad_k, int Cin_pad, const float* __restrict__ bias,
                                                              float* __restrict__ coords, float* __restrict__ flow_out) {
  extern __shared__ __align__(16) uint8_t sm_raw[];
  T* sw = reinterpret_cast<T*>(sm_raw);  // [tap][2][Cin]
  constexpr int TAPS = KH * KW;
  const int c8n = Cin / 8;
  for (int i = threadIdx.x; i < TAPS * 2 * c8n; i += blockDim.x) {
    const int c8 = i % c8n, n = (i / c8n) & 1, tap = i / (2 * c8n);
    reinterpret_cast<uint4*>(sw)[i] = __ldg(reinterpret_cast<const uint4*>(wk + ((size_t)tap * Cout_pad_k + n) * Cin_pad) + c8);
  }
  __syncthreads();
  const int P = B * H * W;
  const int lane = threadIdx.x & 31;
  const int warps_total = gridDim.x * (blockDim.x >> 5);
  const float b0 = bias ? bias[0] : 0.f, b1 = bias ? bias[1] : 0.f;
  for (int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < P; p += warps_total) {
    const int px = p % W, py = (p / W) % H, b = p / (W * H);
    float a0 = 0.f, a1 = 0.f;
    for (int c8 = lane; c8 < c8n; c8 += 32) {
      uint4 xv[TAPS];
#pragma unroll
      for (int tap = 0; tap < TAPS; ++tap) {
        const int iy = py + tap / KW - KH / 2, ix = px + tap % KW - KW / 2;
        const bool inb = iy >= 0 && iy < H && ix >= 0 && ix < W;
        xv[tap] = inb ? __ldg(reinterpret_cast<const uint4*>(x + ((size_t)(b * H + iy) * W + ix) * stride + offset) + c8)
                      : make_uint4(0u, 0u, 0u, 0u);
      }
#pragma unroll
      for (int tap = 0; tap < TAPS; ++tap) {
        float xf[8], f0[8], f1[8];
        unpack8f<T>(xv[tap], xf);
        unpack8f<T>(reinterpret_cast<const uint4*>(sw)[(tap * 2 + 0) * c8n + c8], f0);
        unpack8f<T>(reinterpret_cast<const uint4*>(sw)[(tap * 2 + 1) * c8n + c8], f1);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          a0 = fmaf(xf[e], f0[e], a0);
          a1 = fmaf(xf[e], f1[e], a1);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if (lane == 0) {
      const float c0 = coords[2 * (size_t)p] + a0 + b0;
      const float c1 = coords[2 * (size_t)p + 1] + a1 + b1;
      coords[2 * (size_t)p] = c0;
      coords[2 * (size_t)p + 1] = c1;
      flow_out[2 * (size_t)p] = c0 - (float)px;
      flow_out[2 * (size_t)p + 1] = c1 - (float)py;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// pixel tile FTH x FTW (FTW a multiple of 16); <1,128> gives 440 blocks for the 55x128 grid (one wave at 3 blocks/SM)
template <typename T, int FTH, int FTW>
__global__ void __launch_bounds__(128, 3) conv_flow7x7_kernel(const float* __restrict__ flow, int B, int H, int W,
                                                           const T* __restrict__ w /*[49][2][Cout_pad]*/, int Cout,
                                                           int Cout_pad, const float* __restrict__ bias,
                                                           T* __restrict__ out, int out_stride, int out_offset) {
  pdl_wait();
  pdl_trigger();
  __shared__ float2 patch[FTH + 6][FTW + 6];
  const int PW = (W + FTW - 1) / FTW, PH = (H + FTH - 1) / FTH;
  int t = blockIdx.x;
  const int pw = t % PW;
  t /= PW;
  const int ph = t % PH;
  const int b = t / PH;
  const int x0 = pw * FTW, y0 = ph * FTH;
  for (int i = threadIdx.x; i < (FTH + 6) * (FTW + 6); i += blockDim.x) {
    const int r = i / (FTW + 6), c = i - r * (FTW + 6);
    const int y = y0 + r - 3, x = x0 + c - 3;
    float2 f = make_float2(0.f, 0.f);
    if (y >= 0 && y < H && x >= 0 && x < W) f = *reinterpret_cast<const float2*>(flow + 2 * ((size_t)(b * H + y) * W + x));
    patch[r][c] = f;
  }
  __syncthreads();
  const int n = blockIdx.y * blockDim.x + threadIdx.x;
  if (n >= Cout) return;
  float wr[49][2];
#pragma unroll
  for (int k = 0; k < 49; ++k) {
    wr[k][0] = to_f32(w[(size_t)(k * 2 + 0) * Cout_pad + n]);
    wr[k][1] = to_f32(w[(size_t)(k * 2 + 1) * Cout_pad + n]);
  }
  const float bn = bias ? bias[n] : 0.f;
  for (int ry = 0; ry < FTH; ++ry) {
    const int y = y0 + ry;
    if (y >= H) break;
#pragma unroll 1
    for (int seg = 0; seg < FTW; seg += 16) {
      if (x0 + seg >= W) break;
      float acc[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = bn;
#pragma unroll
      for (int ky = 0; ky < 7; ++ky) {
#pragma unroll
        for (int ix = 0; ix < 16 + 6; ++ix) {
          const float2 v = patch[ry + ky][seg + ix];
#pragma unroll
          for (int kx = 0; kx < 7; ++kx) {
            const int ox = ix - kx;
            if (ox >= 0 && ox < 16) acc[ox] = fmaf(wr[ky * 7 + kx][1], v.y, fmaf(wr[ky * 7 + kx][0], v.x, acc[ox]));
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int x = x0 + seg + i;
        if (x < W) out[((size_t)(b * H + y) * W + x) * out_stride + out_offset + n] = from_f32<T>(fmaxf(acc[i], 0.f));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// delta(p)[o] = bias[o] + sum over the 3x3 neighbourhood of the per-tap products T[p + tap][tap*2 + o]
__global__ void flow_tap_gather_kernel(const float* __restrict__ taps, int tstride, const float* __restrict__ bias,
                                       float* __restrict__ coords, float* __restrict__ flow, int B, int H, int W) {
  pdl_wait();
  pdl_trigger();
  const int P = B * H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int x = p % W, y = (p / W) % H, b = p / (W * H);
  float d0 = bias ? bias[0] : 0.f, d1 = bias ? bias[1] : 0.f;
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int iy = y + tap / 3 - 1, ix = x + tap % 3 - 1;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
      const float2 t = *reinterpret_cast<const float2*>(taps + ((size_t)(b * H + iy) * W + ix) * tstride + 2 * tap);
      d0 += t.x;
      d1 += t.y;
    }
  }
  const float c0 = coords[2 * (size_t)p] + d0, c1 = coords[2 * (size_t)p + 1] + d1;
  coords[2 * (size_t)p] = c0;
  coords[2 * (size_t)p + 1] = c1;
  flow[2 * (size_t)p] = c0 - (float)x;
  flow[2 * (size_t)p + 1] = c1 - (float)y;
}

// ---------------------------------------------------------------------------------------------
struct SrcSplit {
  int n;
  int ch[PFB_MAX_SRC];
};

__global__ void pack_kmajor_kernel(const void* __restrict__ src, void* __restrict__ dst, int Cout, int Cin, int KH, int KW,
                                   int Cout_pad_k, int row_offset, SrcSplit split, int Cin_pad, int sdt, int ddt) {
  const size_t total = (size_t)Cout * Cin * KH * KW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int ci = (int)(idx % Cin);
    size_t t = idx / Cin;
    int co = (int)(t % Cout);
    int tap = (int)(t / Cout);
    // position of input channel ci when every source is padded to a multiple of 64
    int kpos = 0, rem = ci;
    for (int s = 0; s < split.n; ++s) {
      if (rem < split.ch[s]) { kpos += rem; break; }
      rem -= split.ch[s];
      kpos += (split.ch[s] + 63) / 64 * 64;
    }
    float v = load_as_f32(src, ((size_t)co * Cin + ci) * KH * KW + tap, sdt);
    store_from_f32(dst, ((size_t)tap * Cout_pad_k + row_offset + co) * Cin_pad + kpos, ddt, v);
  }
}

// ---------------------------------------------------------------------------------------------
bool conv_cout2_supported(const pfb_conv_params* p) {
  if (p->dtype == PFB_F32 || p->epilogue != PFB_EPI_FLOW || p->Cout != 2 || !p->weight_k) return false;
  if (p->nsrc != 1 || p->src[0].is_f32 || p->KH != 3 || p->KW != 3) return false;
  const pfb_conv_src& s = p->src[0];
  return s.channels % 8 == 0 && s.offset % 8 == 0 && s.stride % 8 == 0 && p->Cin_pad % 8 == 0 && s.channels <= 1024 &&
         (reinterpret_cast<uintptr_t>(s.ptr) & 15) == 0 && p->Cout_pad_k >= 2;
}

int conv_cout2_flow(const pfb_conv_params* p, cudaStream_t s) {
  const int P = p->B * p->H * p->W;
  const pfb_conv_src& x = p->src[0];
  int blocks = ceil_div(P, 8);
  const int cap = sm_count() * 8;
  if (blocks > cap) blocks = cap;
  const size_t smem = (size_t)9 * 2 * x.channels * 2;
  ProfScope prof(KC_CONV, s);
  if (p->dtype == PFB_F16)
    conv_cout2_flow_kernel<__half, 3, 3><<<blocks, 256, smem, s>>>((const __half*)x.ptr, x.stride, x.offset, x.channels, p->B, p->H, p->W,
                                                                   (const __half*)p->weight_k, p->Cout_pad_k, p->Cin_pad, p->bias,
                                                                   p->coords, (float*)p->out);
  else
    conv_cout2_flow_kernel<__nv_bfloat16, 3, 3><<<blocks, 256, smem, s>>>((const __nv_bfloat16*)x.ptr, x.stride, x.offset, x.channels, p->B,
                                                                          p->H, p->W, (const __nv_bfloat16*)p->weight_k, p->Cout_pad_k,
                                                                          p->Cin_pad, p->bias, p->coords, (float*)p->out);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

bool conv_flow7x7_supported(const pfb_conv_params* p) {
  return p->dtype != PFB_F32 && p->nsrc == 1 && p->src[0].is_f32 && p->src[0].channels == 2 && p->src[0].stride == 2 &&
         p->src[0].offset == 0 && p->KH == 7 && p->KW == 7 && p->epilogue == PFB_EPI_RELU;
}

template <typename T, int FTH, int FTW>
static void launch_flow7x7(const pfb_conv_params* p, cudaStream_t s) {
  dim3 grid(ceil_div(p->W, FTW) * ceil_div(p->H, FTH) * p->B, ceil_div(p->Cout, 128));
  launch_pdl(conv_flow7x7_kernel<T, FTH, FTW>, dim3(grid), dim3(128), 0, s, (const float*)p->src[0].ptr, p->B, p->H, p->W, (const T*)p->weight, p->Cout,
                                                        p->Cout_pad, p->bias, (T*)p->out, p->out_stride, p->out_offset);
}

int conv_flow7x7(const pfb_conv_params* p, cudaStream_t s) {
  ProfScope prof(KC_CONV, s);
  const bool rows = (p->W % 128) == 0;  // full-row tiles: no padded columns and a block count that fills whole waves
  if (p->dtype == PFB_F16) {
    if (rows) launch_flow7x7<__half, 1, 128>(p, s); else launch_flow7x7<__half, 8, 16>(p, s);
  } else {
    if (rows) launch_flow7x7<__nv_bfloat16, 1, 128>(p, s); else launch_flow7x7<__nv_bfloat16, 8, 16>(p, s);
  }
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_pack_conv_weight_kmajor(const void* src, void* dst, int Cout, int Cin, int KH, int KW,
                                                   int Cout_pad_k, int row_offset, const int* src_channels, int nsrc,
                                                   int Cin_pad, pfb_dtype src_dtype, pfb_dtype dst_dtype, pfb_stream stream) {
  PFB_CHECK_ARG(src && dst && src_channels, "pack_conv_weight_kmajor: null pointer");
  PFB_CHECK_ARG(dtype_ok(src_dtype) && dtype_ok(dst_dtype), "pack_conv_weight_kmajor: bad dtype");
  PFB_CHECK_ARG(nsrc >= 1 && nsrc <= PFB_MAX_SRC, "pack_conv_weight_kmajor: nsrc=%d", nsrc);
  PFB_CHECK_ARG(Cout > 0 && Cin > 0 && KH > 0 && KW > 0 && row_offset >= 0 && row_offset + Cout <= Cout_pad_k,
                "pack_conv_weight_kmajor: bad shape");
  SrcSplit sp{};
  sp.n = nsrc;
  int sum = 0, padded = 0;
  for (int i = 0; i < nsrc; ++i) {
    PFB_CHECK_ARG(src_channels[i] > 0, "pack_conv_weight_kmajor: source %d has %d channels", i, src_channels[i]);
    sp.ch[i] = src_channels[i];
    sum += src_channels[i];
    padded += (src_channels[i] + 63) / 64 * 64;
  }
  PFB_CHECK_ARG(sum == Cin && padded == Cin_pad, "pack_conv_weight_kmajor: sources sum to %d (pad %d), expected Cin=%d Cin_pad=%d", sum,
                padded, Cin, Cin_pad);
  size_t total = (size_t)Cout * Cin * KH * KW;
  unsigned blocks = (unsigned)(ceil_div_sz(total, 256) > 4096 ? 4096 : ceil_div_sz(total, 256));
  ProfScope prof(KC_MISC, as_stream(stream));
  pack_kmajor_kernel<<<blocks, 256, 0, as_stream(stream)>>>(src, dst, Cout, Cin, KH, KW, Cout_pad_k, row_offset, sp, Cin_pad,
                                                            (int)src_dtype, (int)dst_dtype);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_flow_tap_gather(const float* taps, int tstride, const float* bias, float* coords, float* flow, int B, int H,
                                           int W, pfb_stream stream) {
  PFB_CHECK_ARG(taps && coords && flow && B > 0 && H > 0 && W > 0 && tstride >= 18 && tstride % 2 == 0, "flow_tap_gather: bad arguments");
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_GATHER, s);
  launch_pdl(flow_tap_gather_kernel, dim3(ceil_div(B * H * W, 256)), dim3(256), 0, s, taps, tstride, bias, coords, flow, B, H, W);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
