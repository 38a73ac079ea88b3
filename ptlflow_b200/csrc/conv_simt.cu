// Generic stride-1 "same" convolution as an implicit GEMM on the CUDA cores, fp32 accumulate.
// This is the reference-precision path (fp32 parity <= 1e-3, raft_small, odd channel counts);
// the f16/bf16 production path is conv_umma.cu (wgmma).  It evaluates the reference's
// nn.Conv2d + activation (+ GRU gate arithmetic) of ptlflow/models/raft/update.py:6-153
// without materialising any torch.cat: the K loop walks (tap, source, channel-chunk).
#include "common.cuh"

namespace pfb {

struct SrcDev {
  const void* ptr;
  int channels, stride, offset, is_f32;
};

struct ConvDev {
  SrcDev src[PFB_MAX_SRC];
  int nsrc;
  int B, H, W, KH, KW;
  int Cin_total, Cout, Cout_pad;
  const void* weight;
  const float* bias;
  int epilogue;
  float scale;
  void* out;
  int out_stride, out_offset;
  const void* aux_h;
  void* aux_z;
  int hidden;
  float* coords;
  const float* flow;
  const void* residual;
  int residual_stride, residual_offset;
  const float* post_w;
  const float* post_b;
};

template <typename T>
__device__ __forceinline__ float load_src(const SrcDev& s, size_t pix, int c) {
  size_t i = pix * s.stride + s.offset + c;
  if (s.is_f32) return reinterpret_cast<const float*>(s.ptr)[i];
  return to_f32(reinterpret_cast<const T*>(s.ptr)[i]);
}

// Position of a K chunk: (tap, source, first channel).  The K loop walks taps outermost, then the concatenated sources,
// then 32-channel chunks -- the order of the weight rows ((tap * Cin_total + channel) * Cout_pad).
struct KPos {
  int tap, s, c0, cbase;  // cbase = weight row of channel 0 of source s at this tap
};

// BM x 64 output tile per CTA (BM = 64 / 32 / 16 pixels: the smaller tiles are for small images, where 64-pixel tiles
// leave most SMs without a CTA), 32-deep K chunks.  The next chunk's operands are fetched into registers while the current
// one is multiplied out of shared memory (double-buffered, one barrier per chunk): the first version loaded, synchronised,
// multiplied and synchronised again per 16-deep chunk, i.e. it paid the global-memory latency K / 16 times in sequence --
// 97 us per layer at raft_small's 16 x 32 grid (BASELINE config 1), whatever the number of CTAs.  The accumulation order
// along K is unchanged (ascending, one fma per element), so results are bit-identical to that version.
template <typename T, int BM>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvDev a) {
  constexpr int BN = 64, BK = 32;
  constexpr int MI = BM / 16;           // output pixels per thread (x 4 output channels)
  constexpr int AV = BM * BK / 256;     // A values per thread and chunk: 8 / 4 / 2 consecutive channels of one pixel
  constexpr int TPP = BK / AV;          // threads per pixel in the A loader
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  const int P = a.B * a.H * a.W;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int ml = tid / TPP, kq = (tid % TPP) * AV;   // A loader: pixel ml, AV consecutive channels starting at kq
  const int kb = tid >> 4, nq = (tid & 15) * 4;       // B loader: k rows kb and kb + 16, 4 consecutive output channels at nq
  const int pl = m0 + ml;
  int lb = 0, ly = 0, lx = 0;
  const bool pvalid = pl < P;
  if (pvalid) {
    lx = pl % a.W;
    int t = pl / a.W;
    ly = t % a.H;
    lb = t / a.H;
  }
  const int ph = a.KH / 2, pw = a.KW / 2;
  const int ntaps = a.KH * a.KW;
  const T* wgt = reinterpret_cast<const T*>(a.weight);
  float acc[MI][4] = {};
  float ra[AV], rb[8];

  auto fetch = [&](const KPos& k) {  // global -> registers (no use of the values here: the loads stay in flight)
    const int ky = k.tap / a.KW, kx = k.tap - ky * a.KW;
    const int iy = ly + ky - ph, ix = lx + kx - pw;
    const bool inb = pvalid && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
    const size_t ipix = ((size_t)lb * a.H + (inb ? iy : 0)) * a.W + (inb ? ix : 0);
    const SrcDev& src = a.src[k.s];
#pragma unroll
    for (int j = 0; j < AV; ++j) {
      const int c = k.c0 + kq + j;
      ra[j] = (inb && c < src.channels) ? load_src<T>(src, ipix, c) : 0.f;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = k.c0 + kb + 16 * h;
      const bool kval = c < src.channels;
      const T* wrow = wgt + (size_t)(k.cbase + (kval ? c : 0)) * a.Cout_pad;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + nq + j;
        rb[4 * h + j] = (kval && n < a.Cout_pad) ? to_f32(wrow[n]) : 0.f;
      }
    }
  };
  auto stash = [&](int buf) {  // registers -> shared memory
#pragma unroll
    for (int j = 0; j < AV; ++j) As[buf][kq + j][ml] = ra[j];
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float4*>(&Bs[buf][kb + 16 * h][nq]) = make_float4(rb[4 * h], rb[4 * h + 1], rb[4 * h + 2], rb[4 * h + 3]);
  };
  auto advance = [&](KPos& k) -> bool {  // next chunk; false after the last one
    k.c0 += BK;
    if (k.c0 >= a.src[k.s].channels) {
      k.c0 = 0;
      k.cbase += a.src[k.s].channels;
      if (++k.s == a.nsrc) {
        k.s = 0;
        ++k.tap;  // cbase has advanced by Cin_total = the next tap's first row
      }
    }
    return k.tap < ntaps;
  };

  KPos k{0, 0, 0, 0};
  fetch(k);
  stash(0);
  __syncthreads();
  int buf = 0;
  bool more = advance(k);
  while (true) {
    if (more) fetch(k);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float av[MI];
      if (MI == 4) {
        const float4 v = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
        av[0] = v.x; av[1 % MI] = v.y; av[2 % MI] = v.z; av[3 % MI] = v.w;
      } else if (MI == 2) {
        const float2 v = *reinterpret_cast<const float2*>(&As[buf][kk][ty * 2]);
        av[0] = v.x; av[1 % MI] = v.y;
      } else {
        av[0] = As[buf][kk][ty];
      }
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
#pragma unroll
      for (int i = 0; i < MI; ++i) {
        acc[i][0] = fmaf(av[i], bv.x, acc[i][0]);
        acc[i][1] = fmaf(av[i], bv.y, acc[i][1]);
        acc[i][2] = fmaf(av[i], bv.z, acc[i][2]);
        acc[i][3] = fmaf(av[i], bv.w, acc[i][3]);
      }
    }
    if (!more) break;
    stash(buf ^ 1);  // the other buffer was last read before the previous barrier
    __syncthreads();
    buf ^= 1;
    more = advance(k);
  }

  // ---- epilogue --------------------------------------------------------------------------
  const int hd = a.hidden;
#pragma unroll
  for (int i = 0; i < MI; ++i) {
    const int p = m0 + ty * MI + i;
    if (p >= P) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= a.Cout) continue;
      float v = acc[i][j] + (a.bias ? a.bias[n] : 0.f);
      switch (a.epilogue) {
        case PFB_EPI_LINEAR:
          reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = from_f32<T>(v * a.scale);
          break;
        case PFB_EPI_RELU:
        case PFB_EPI_RELU_APPEND_FLOW:
          reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = from_f32<T>(fmaxf(v, 0.f));
          break;
        case PFB_EPI_LINEAR_APPEND_FLOW:
          reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = from_f32<T>(v);
          break;
        case PFB_EPI_GELU:
          reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = from_f32<T>(gelu_f32(v));
          break;
        case PFB_EPI_RESIDUAL_GELU: {
          const float res = to_f32(reinterpret_cast<const T*>(a.residual)[(size_t)p * a.residual_stride + a.residual_offset + n]);
          float y = gelu_f32(res + v);
          if (a.post_w) y = gelu_f32(fmaf(y, 1.f + a.post_w[n], a.post_b[n]));
          reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = from_f32<T>(y);
          break;
        }
        case PFB_EPI_GRU_ZR: {
          float g = sigmoid_f32(v);
          if (n < hd) {
            reinterpret_cast<T*>(a.aux_z)[(size_t)p * hd + n] = from_f32<T>(g);
          } else {
            float h = to_f32(reinterpret_cast<const T*>(a.aux_h)[(size_t)p * hd + (n - hd)]);
            reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + (n - hd)] = from_f32<T>(g * h);
          }
          break;
        }
        case PFB_EPI_GRU_Q: {
          float q = tanhf(v);
          float z = to_f32(reinterpret_cast<const T*>(a.aux_z)[(size_t)p * hd + n]);
          float h = to_f32(reinterpret_cast<const T*>(a.aux_h)[(size_t)p * hd + n]);
          reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = from_f32<T>((1.f - z) * h + z * q);
          break;
        }
        case PFB_EPI_LINEAR_F32:
          reinterpret_cast<float*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = v * a.scale;
          break;
        case PFB_EPI_AXPY: {
          float res = to_f32(reinterpret_cast<const T*>(a.aux_h)[(size_t)p * hd + n]);
          reinterpret_cast<T*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = from_f32<T>(res + a.scale * v);
          break;
        }
        case PFB_EPI_FLOW: {
          // n in {0,1}: coords1 += delta ; flow = coords1 - coords0, coords0 = (x, y)
          float c1 = a.coords[(size_t)p * 2 + n] + v;
          a.coords[(size_t)p * 2 + n] = c1;
          int x = p % a.W, y = (p / a.W) % a.H;
          reinterpret_cast<float*>(a.out)[(size_t)p * a.out_stride + a.out_offset + n] = c1 - (float)(n == 0 ? x : y);
          break;
        }
        default:
          break;
      }
    }
    if ((a.epilogue == PFB_EPI_RELU_APPEND_FLOW || a.epilogue == PFB_EPI_LINEAR_APPEND_FLOW) && blockIdx.y == 0 && tx == 0) {
      T* o = reinterpret_cast<T*>(a.out) + (size_t)p * a.out_stride + a.out_offset + a.Cout;
      o[0] = from_f32<T>(a.flow[(size_t)p * 2]);
      o[1] = from_f32<T>(a.flow[(size_t)p * 2 + 1]);
    }
  }
}

int conv2d_simt(const pfb_conv_params* p, cudaStream_t s) {
  ConvDev a;
  a.nsrc = p->nsrc;
  int cin = 0;
  for (int i = 0; i < p->nsrc; ++i) {
    a.src[i].ptr = p->src[i].ptr;
    a.src[i].channels = p->src[i].channels;
    a.src[i].stride = p->src[i].stride;
    a.src[i].offset = p->src[i].offset;
    a.src[i].is_f32 = p->src[i].is_f32 || p->dtype == PFB_F32;
    cin += p->src[i].channels;
  }
  a.B = p->B; a.H = p->H; a.W = p->W; a.KH = p->KH; a.KW = p->KW;
  a.Cin_total = cin; a.Cout = p->Cout; a.Cout_pad = p->Cout_pad;
  a.weight = p->weight; a.bias = p->bias; a.epilogue = p->epilogue; a.scale = p->scale;
  a.out = p->out; a.out_stride = p->out_stride; a.out_offset = p->out_offset;
  a.aux_h = p->aux_h; a.aux_z = p->aux_z; a.hidden = p->hidden; a.coords = p->coords; a.flow = p->flow;
  a.residual = p->residual; a.residual_stride = p->residual_stride; a.residual_offset = p->residual_offset;
  a.post_w = p->post_w; a.post_b = p->post_b;
  const int P = p->B * p->H * p->W;
  // small images: smaller pixel tiles until the grid covers the machine (each CTA's K loop is a latency chain)
  const int n_tiles = ceil_div(p->Cout, 64), sms = sm_count();
  const int bm = ceil_div(P, 64) * n_tiles >= sms ? 64 : (ceil_div(P, 32) * n_tiles >= sms ? 32 : 16);
  dim3 grid(ceil_div(P, bm), n_tiles);
  {
    ProfScope prof(KC_CONV, s);
    if (bm == 64) PFB_DISPATCH_DTYPE(p->dtype, T, { conv_simt_kernel<T, 64><<<grid, 256, 0, s>>>(a); });
    else if (bm == 32) PFB_DISPATCH_DTYPE(p->dtype, T, { conv_simt_kernel<T, 32><<<grid, 256, 0, s>>>(a); });
    else PFB_DISPATCH_DTYPE(p->dtype, T, { conv_simt_kernel<T, 16><<<grid, 256, 0, s>>>(a); });
  }
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_conv2d(const pfb_conv_params* p, pfb_stream stream) {
  PFB_CHECK_ARG(p, "conv2d: null params");
  PFB_CHECK_ARG(dtype_ok(p->dtype), "conv2d: bad dtype %d", (int)p->dtype);
  PFB_CHECK_ARG(p->nsrc >= 1 && p->nsrc <= PFB_MAX_SRC, "conv2d: nsrc=%d out of range", p->nsrc);
  PFB_CHECK_ARG(p->B > 0 && p->H > 0 && p->W > 0, "conv2d: bad shape");
  PFB_CHECK_ARG((p->KH & 1) && (p->KW & 1) && p->KH <= 15 && p->KW <= 15, "conv2d: kernel %dx%d must be odd", p->KH, p->KW);
  PFB_CHECK_ARG(p->Cout > 0 && p->Cout_pad >= p->Cout, "conv2d: Cout=%d Cout_pad=%d", p->Cout, p->Cout_pad);
  PFB_CHECK_ARG(p->weight && p->out, "conv2d: null weight/out");
  for (int i = 0; i < p->nsrc; ++i) {
    PFB_CHECK_ARG(p->src[i].ptr && p->src[i].channels > 0 && p->src[i].stride >= p->src[i].offset + p->src[i].channels,
                  "conv2d: bad source %d", i);
  }
  switch (p->epilogue) {
    case PFB_EPI_LINEAR: case PFB_EPI_RELU: case PFB_EPI_LINEAR_F32: case PFB_EPI_GELU: break;
    case PFB_EPI_RESIDUAL_GELU:
      PFB_CHECK_ARG(p->residual && p->residual_stride >= p->residual_offset + p->Cout && p->residual_offset >= 0,
                    "conv2d: RESIDUAL_GELU needs a residual with stride >= offset + Cout");
      PFB_CHECK_ARG((p->post_w == nullptr) == (p->post_b == nullptr), "conv2d: RESIDUAL_GELU needs both post_w and post_b, or neither");
      break;
    case PFB_EPI_AXPY:
      PFB_CHECK_ARG(p->aux_h && p->hidden >= p->Cout, "conv2d: AXPY needs aux_h (residual) with stride hidden >= Cout");
      break;
    case PFB_EPI_GRU_ZR:
      PFB_CHECK_ARG(p->aux_h && p->aux_z && p->hidden > 0 && p->Cout == 2 * p->hidden, "conv2d: GRU_ZR needs aux_h, aux_z and Cout == 2*hidden");
      break;
    case PFB_EPI_GRU_Q:
      PFB_CHECK_ARG(p->aux_h && p->aux_z && p->hidden > 0 && p->Cout == p->hidden, "conv2d: GRU_Q needs aux_h, aux_z and Cout == hidden");
      break;
    case PFB_EPI_FLOW:
      PFB_CHECK_ARG(p->coords && p->Cout == 2, "conv2d: FLOW epilogue needs coords and Cout == 2");
      break;
    case PFB_EPI_RELU_APPEND_FLOW:
    case PFB_EPI_LINEAR_APPEND_FLOW:
      PFB_CHECK_ARG(p->flow && p->out_stride >= p->out_offset + p->Cout + 2, "conv2d: APPEND_FLOW needs flow and room for 2 channels");
      break;
    default:
      set_error("conv2d: unknown epilogue %d", p->epilogue);
      return PFB_ERR_ARG;
  }
  cudaStream_t s = as_stream(stream);
  if (p->impl != 1) {
    if (conv_cout2_supported(p)) return conv_cout2_flow(p, s);
    if (conv_flow7x7_supported(p)) return conv_flow7x7(p, s);
    if (conv2d_umma_supported(p)) return conv2d_umma(p, s);
    if (p->impl == 2) {
      set_error("conv2d: wgmma path does not support this shape/dtype");
      return PFB_ERR_UNSUPPORTED;
    }
  }
  if (p->addend || p->w_rows_per_sample) {
    set_error("conv2d: per-pixel addend / per-sample weights are implemented by the wgmma path only (shape / dtype / impl not eligible)");
    return PFB_ERR_UNSUPPORTED;
  }
  return conv2d_simt(p, s);
}
