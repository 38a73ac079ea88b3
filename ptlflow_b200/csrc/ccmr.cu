// CCMR's XCiT global context (ptlflow/models/ccmr/xcit.py:58-427) on top of the ms_raft_plus scale loop: the Fourier positional
// features, the XCA statistics and their fold into one per-sample linear layer, the residual-stream set-up, the whole XCABlock as
// a launch sequence, and the bilinear upflow2 of the output (ccmr/utils.py:97-99).
//
// The fold (DESIGN.md section 1, row a18): in XCA, q and k are L2-normalised over the N pixels and A_h = softmax(t_h q^ k^T) is a
// 16 x 16 matrix per head, so proj(A v) = W_proj blockdiag(A) W_v LN1(x_v) + bias is one 128 x 128 linear of LN1(x_v) per sample.
// For the aggregator, q and k come from the scale's global context only: its A is a constant of the scale, and each iteration's
// attention is one GEMM with per-sample weights whose epilogue adds the residual stream (global_context + pos + folded bias).
#include <algorithm>
#include <atomic>

#include "refine.cuh"

#define PFB_TRY(expr)        \
  do {                       \
    int rc__ = (expr);       \
    if (rc__ != PFB_OK) return rc__; \
  } while (0)

namespace pfb {

constexpr int kXcaC = 128, kXcaHeads = 8, kXcaD = 16;
constexpr int kXcaStats = kXcaHeads * kXcaD * kXcaD + 2 * kXcaC;  // 2048 gram entries + 256 sums of squares
constexpr int kXcaChunk = 512;                                    // pixels per statistics CTA (fixed: the combine order is fixed)
constexpr int kXcaTile = 32;                                      // pixels staged per step

// PositionalEncodingFourier.forward before token_projection (xcit.py:73-93), in fp32 like the reference's fp32 model
template <typename T>
__global__ void fourier_features_kernel(T* __restrict__ out, int H, int W) {
  const size_t total = (size_t)H * W * 64;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(idx % 64);
    const size_t p = idx / 64;
    const int x = (int)(p % W), y = (int)(p / W);
    const int d = ch & 31;
    // y_embed = cumsum / (last + eps) * 2 pi;  dim_t = 10000 ** (2 * (d // 2) / 32)
    const float e = ch < 32 ? (float)(y + 1) / ((float)H + 1e-6f) * 6.2831855f : (float)(x + 1) / ((float)W + 1e-6f) * 6.2831855f;
    const float dim_t = powf(10000.f, (2.f * (float)(d / 2)) / 32.f);
    const float a = e / dim_t;
    out[idx] = from_f32<T>((d & 1) ? cosf(a) : sinf(a));
  }
}

// Per (sample, chunk of kXcaChunk pixels): fp32 partial gram of every head and sums of squares of q and k.  Thread t owns gram
// entries (h = t / 32, i = (t / 2) % 16, j = 8 (t % 2) .. +7) and the sum of squares of column t of [q | k].
template <typename T>
__global__ void __launch_bounds__(256) xca_stats_kernel(const T* __restrict__ qk, int stride, int q_off, int k_off, int N, int chunks,
                                                        float* __restrict__ partial) {
  __shared__ float s_qk[kXcaTile][2 * kXcaC + 1];
  const int b = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const int h = tid >> 5, i = (tid >> 1) & 15, j0 = (tid & 1) * 8;
  const int qc = h * kXcaD + i, kc = kXcaC + h * kXcaD + j0;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, ss = 0.f;
  const int n0 = chunk * kXcaChunk, n1 = min(N, n0 + kXcaChunk);
  const T* base = qk + (size_t)b * N * stride;
  for (int t0 = n0; t0 < n1; t0 += kXcaTile) {
    for (int e = tid; e < kXcaTile * 2 * kXcaC; e += 256) {
      const int px = e / (2 * kXcaC), c = e % (2 * kXcaC), n = t0 + px;
      float v = 0.f;
      if (n < n1) v = to_f32(base[(size_t)n * stride + (c < kXcaC ? q_off + c : k_off + c - kXcaC)]);
      s_qk[px][c] = v;
    }
    __syncthreads();
#pragma unroll 4
    for (int px = 0; px < kXcaTile; ++px) {
      const float q = s_qk[px][qc];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) acc[jj] = fmaf(q, s_qk[px][kc + jj], acc[jj]);
      const float v = s_qk[px][tid];
      ss = fmaf(v, v, ss);
    }
    __syncthreads();
  }
  float* o = partial + ((size_t)b * chunks + chunk) * kXcaStats;
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) o[h * 256 + i * 16 + j0 + jj] = acc[jj];
  o[2048 + tid] = ss;
}

// stats[b][e] = sum over the chunks, in chunk order, in fp64
__global__ void xca_combine_kernel(const float* __restrict__ partial, int chunks, float* __restrict__ stats) {
  const int b = blockIdx.y, e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= kXcaStats) return;
  const float* p = partial + (size_t)b * chunks * kXcaStats + e;
  double s = 0.0;
  for (int c = 0; c < chunks; ++c) s += (double)p[(size_t)c * kXcaStats];
  stats[(size_t)b * kXcaStats + e] = (float)s;
}

// grid (B, 8 blocks of 16 output rows), 256 threads.  A (fp32 softmax), M = blockdiag(A) v_w and m_b = blockdiag(A) v_b in shared
// memory, then rows o of W = proj_w M and bias = proj_w m_b + proj_b.
constexpr size_t kFoldSmem = (size_t)(kXcaHeads * kXcaD * kXcaD + kXcaC * kXcaC + kXcaC) * sizeof(float);

template <typename T>
__global__ void __launch_bounds__(256) xca_fold_kernel(const float* __restrict__ stats, const float* __restrict__ temperature,
                                                       const float* __restrict__ v_w, const float* __restrict__ v_b,
                                                       const float* __restrict__ proj_w, const float* __restrict__ proj_b,
                                                       T* __restrict__ w_out, T* __restrict__ w_out_k, float* __restrict__ bias_out) {
  extern __shared__ float fold_sm[];
  float* sA = fold_sm;                                  // [8][16][16]
  float* sM = sA + kXcaHeads * kXcaD * kXcaD;           // [128][128]
  float* sm = sM + kXcaC * kXcaC;                       // [128]
  const int b = blockIdx.x, ob = blockIdx.y, tid = threadIdx.x;
  const float* st = stats + (size_t)b * kXcaStats;
  if (tid < kXcaC) {  // row (h, i) of A
    const int h = tid / kXcaD;
    const float nq = fmaxf(sqrtf(st[2048 + tid]), 1e-12f), t = temperature[h];
    float l[kXcaD], mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < kXcaD; ++j) {
      const float nk = fmaxf(sqrtf(st[2176 + h * kXcaD + j]), 1e-12f);
      l[j] = (st[h * 256 + (tid % kXcaD) * 16 + j] / (nq * nk)) * t;
      mx = fmaxf(mx, l[j]);
    }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < kXcaD; ++j) {
      l[j] = expf(l[j] - mx);
      sum += l[j];
    }
#pragma unroll
    for (int j = 0; j < kXcaD; ++j) sA[tid * kXcaD + j] = l[j] / sum;
  }
  __syncthreads();
  for (int e = tid; e < kXcaC * kXcaC; e += 256) {
    const int c = e / kXcaC, i = e % kXcaC, h = c / kXcaD;
    const float* a = sA + c * kXcaD;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < kXcaD; ++j) acc = fmaf(a[j], __ldg(v_w + (size_t)(h * kXcaD + j) * kXcaC + i), acc);
    sM[e] = acc;
  }
  if (tid < kXcaC) {
    const int h = tid / kXcaD;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < kXcaD; ++j) acc = fmaf(sA[tid * kXcaD + j], v_b[h * kXcaD + j], acc);
    sm[tid] = acc;
  }
  __syncthreads();
  for (int e = tid; e < 16 * kXcaC; e += 256) {
    const int o = ob * 16 + e / kXcaC, i = e % kXcaC;
    const float* pw = proj_w + (size_t)o * kXcaC;
    float acc = 0.f;
    for (int c = 0; c < kXcaC; ++c) acc = fmaf(__ldg(pw + c), sM[c * kXcaC + i], acc);
    const T v = from_f32<T>(acc);
    w_out[((size_t)b * kXcaC + i) * kXcaC + o] = v;
    if (w_out_k) w_out_k[((size_t)b * kXcaC + o) * kXcaC + i] = v;
  }
  if (tid < 16) {
    const int o = ob * 16 + tid;
    const float* pw = proj_w + (size_t)o * kXcaC;
    float acc = proj_b[o];
    for (int c = 0; c < kXcaC; ++c) acc = fmaf(pw[c], sm[c], acc);
    bias_out[(size_t)b * kXcaC + o] = acc;
  }
}

// out[b, n, c] = a[b, n, a_offset + c] + (pos ? pos[n, c] : 0) + (vec ? vec[b, c] : 0), C = 128, out stride 128; fp32 sum, one rounding
template <typename T>
__global__ void xcit_residual_kernel(const T* __restrict__ a, int a_stride, const T* __restrict__ pos, const float* __restrict__ vec,
                                     T* __restrict__ out, int B, int N) {
  const size_t total = (size_t)B * N * kXcaC;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % kXcaC);
    const size_t p = idx / kXcaC;
    const int n = (int)(p % N), b = (int)(p / N);
    float v = to_f32(a[p * a_stride + c]);
    if (pos) v += to_f32(pos[(size_t)n * kXcaC + c]);
    if (vec) v += vec[(size_t)b * kXcaC + c];
    out[idx] = from_f32<T>(v);
  }
}

// upflow2: 2 * F.interpolate(flow, 2x, bilinear, align_corners=True), with ATen's fp32 source index arithmetic
__global__ void upflow2_kernel(const float* __restrict__ flow, float* __restrict__ out, int B, int H, int W, int OH, int OW, int pad_top,
                               int pad_left) {
  const int FH = 2 * H, FW = 2 * W;
  const float rh = FH > 1 ? (float)(H - 1) / (float)(FH - 1) : 0.f, rw = FW > 1 ? (float)(W - 1) / (float)(FW - 1) : 0.f;
  const size_t total = (size_t)B * OH * OW;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % OW);
    const size_t t = idx / OW;
    const int oy = (int)(t % OH), b = (int)(t / OH);
    const float fy = rh * (float)(oy + pad_top), fx = rw * (float)(ox + pad_left);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < H - 1 ? 1 : 0), x1 = x0 + (x0 < W - 1 ? 1 : 0);
    const float ly = fy - (float)y0, lx = fx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float* f = flow + (size_t)(b * 2 + c) * H * W;
      const float v = hy * (hx * f[(size_t)y0 * W + x0] + lx * f[(size_t)y0 * W + x1]) +
                      ly * (hx * f[(size_t)y1 * W + x0] + lx * f[(size_t)y1 * W + x1]);
      out[((size_t)(b * 2 + c) * OH + oy) * OW + ox] = 2.f * v;
    }
  }
}

static unsigned grid_for(size_t total, int per_sm = 16) {
  return (unsigned)std::max<size_t>(1, std::min<size_t>(ceil_div_sz(total, 256), (size_t)sm_count() * per_sm));
}

static int xcit_residual(const void* a, int a_stride, const void* pos, const float* vec, void* out, int B, int N, pfb_dtype dt,
                         cudaStream_t s) {
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dt, T, {
    xcit_residual_kernel<T><<<grid_for((size_t)B * N * kXcaC), 256, 0, s>>>((const T*)a, a_stride, (const T*)pos, vec, (T*)out, B, N);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

// ---- the scale's workspace (after the update loop's own, see refine.cu) ----
CcmrPlan ccmr_plan(const pfb_raft_cfg* c) {
  CcmrPlan w{};
  const size_t N = (size_t)c->H * c->W, P = (size_t)c->B * N, es = dtype_size(c->dtype), row = kXcaC * es;
  w.chunks = (int)ceil_div_sz(N, kXcaChunk);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  w.off_feat = take(N * 64 * es);
  w.off_pos_c = take(N * row);
  w.off_pos_a = take(N * row);
  w.off_x0 = take(P * row);
  w.off_ln = take(P * row);
  w.off_qk = take(P * 2 * row);
  w.off_x1 = take(P * row);
  w.off_t = take(P * row);
  w.off_u = take(P * row);
  w.off_gc = take(P * row);
  w.off_wf = take((size_t)c->B * kXcaC * row);
  w.off_wfk = take((size_t)c->B * kXcaC * row);
  w.off_bf = take((size_t)c->B * kXcaC * sizeof(float));
  w.off_part = take((size_t)c->B * w.chunks * kXcaStats * sizeof(float));
  w.off_stats = take((size_t)c->B * kXcaStats * sizeof(float));
  w.off_gn = take(pfb_instance_norm_workspace_bytes(c->B, kXcaC));
  w.off_up = take(P * 4 * 2 * sizeof(float));  // the padded 2x flow ahead of upflow2
  w.total = off;
  return w;
}

struct Xs {  // one scale's buffers
  const pfb_raft_cfg* c;
  CcmrPlan pl;
  char* base;
  cudaStream_t s;
  void* at(size_t off) const { return base + off; }
};

static int conv1x1s(const Xs& x, const pfb_layer& L, int B, int H, int W, const void* src, int src_stride, int src_offset, int epi, void* out,
                    int out_stride, int out_offset, const void* aux = nullptr, int aux_stride = 0) {
  pfb_conv_params p{};
  PFB_CHECK_ARG(L.weight && L.KH == 1 && L.KW == 1, "ccmr: missing 1x1 layer");
  p.src[0].ptr = src; p.src[0].channels = L.Cin; p.src[0].stride = src_stride; p.src[0].offset = src_offset; p.src[0].is_f32 = 0;
  p.nsrc = 1;
  p.B = B; p.H = H; p.W = W; p.KH = 1; p.KW = 1;
  p.Cout = L.Cout; p.Cout_pad = L.Cout_pad; p.weight = L.weight; p.bias = L.bias;
  p.epilogue = epi; p.scale = 1.f;
  p.out = out; p.out_stride = out_stride; p.out_offset = out_offset;
  p.aux_h = aux; p.hidden = aux_stride;
  p.dtype = x.c->dtype; p.impl = x.c->impl;
  p.weight_k = L.weight_k; p.Cin_pad = L.Cin_pad; p.Cout_pad_k = L.Cout_pad_k;
  return pfb_conv2d(&p, (pfb_stream)x.s);
}

// x0 (the block's residual stream, [P][128]) -> ln = LN1(x0) without affine, the folded attention (wf, wfk, bf) and, in place,
// x0 + bf: the addend of the attention GEMM
static int xcit_prepare(const Xs& x, const pfb_xcit_block& w) {
  const pfb_raft_cfg* c = x.c;
  const int N = c->H * c->W;
  const size_t P = (size_t)c->B * N;
  void* x0 = x.at(x.pl.off_x0);
  void* ln = x.at(x.pl.off_ln);
  void* qk = x.at(x.pl.off_qk);
  float* stats = reinterpret_cast<float*>(x.at(x.pl.off_stats));
  float* bf = reinterpret_cast<float*>(x.at(x.pl.off_bf));
  PFB_CHECK_ARG(w.qk.Cin == kXcaC && w.qk.Cout == 2 * kXcaC, "ccmr: the q | k layer must be 128 -> 256");
  PFB_CHECK_ARG(w.v_weight && w.v_bias && w.proj_weight && w.proj_bias && w.temperature, "ccmr: null XCA weights");
  PFB_TRY(pfb_layernorm(x0, kXcaC, 0, ln, kXcaC, 0, nullptr, nullptr, P, kXcaC, w.ln_eps, c->dtype, (pfb_stream)x.s));
  PFB_TRY(conv1x1s(x, w.qk, c->B, c->H, c->W, ln, kXcaC, 0, PFB_EPI_LINEAR, qk, 2 * kXcaC, 0));
  PFB_TRY(pfb_xca_stats(qk, 2 * kXcaC, 0, kXcaC, c->B, N, stats, x.at(x.pl.off_part), c->dtype, (pfb_stream)x.s));
  const bool kmajor = c->dtype != PFB_F32;
  PFB_TRY(pfb_xca_fold(stats, w.temperature, w.v_weight, w.v_bias, w.proj_weight, w.proj_bias, x.at(x.pl.off_wf),
                       kmajor ? x.at(x.pl.off_wfk) : nullptr, bf, c->B, c->dtype, (pfb_stream)x.s));
  return xcit_residual(x0, kXcaC, nullptr, bf, x0, c->B, N, c->dtype, x.s);
}

// out[:, out_offset .. +127] = block(x0) given v_ln = LN1(x_v) without affine (xcit.py:291-300), after xcit_prepare
static int xcit_apply(const Xs& x, const pfb_xcit_block& w, const void* v_ln, void* out, int out_stride, int out_offset) {
  const pfb_raft_cfg* c = x.c;
  const int N = c->H * c->W;
  const size_t P = (size_t)c->B * N, es = dtype_size(c->dtype);
  const pfb_stream st = (pfb_stream)x.s;
  void* add = x.at(x.pl.off_x0);
  void* x1 = x.at(x.pl.off_x1);
  void* t = x.at(x.pl.off_t);
  void* u = x.at(x.pl.off_u);
  // x1 = x0 + gamma1 * proj(A v): per-sample folded weights, the residual (with the folded bias) in the AXPY epilogue
  const char* wf = reinterpret_cast<const char*>(x.at(x.pl.off_wf));
  if (c->dtype != PFB_F32 && c->impl != 1) {
    pfb_conv_params p{};
    p.src[0].ptr = v_ln; p.src[0].channels = kXcaC; p.src[0].stride = kXcaC;
    p.nsrc = 1;
    p.B = c->B; p.H = c->H; p.W = c->W; p.KH = 1; p.KW = 1;
    p.Cout = kXcaC; p.Cout_pad = kXcaC; p.weight = wf; p.bias = nullptr;
    p.epilogue = PFB_EPI_AXPY; p.scale = 1.f;
    p.out = x1; p.out_stride = kXcaC; p.out_offset = 0;
    p.aux_h = add; p.hidden = kXcaC;
    p.dtype = c->dtype; p.impl = 2;
    p.weight_k = x.at(x.pl.off_wfk); p.Cin_pad = kXcaC; p.Cout_pad_k = kXcaC;
    p.w_rows_per_sample = kXcaC;
    PFB_TRY(pfb_conv2d(&p, st));
  } else {
    for (int b = 0; b < c->B; ++b) {  // SIMT: one launch per sample with that sample's weights
      const size_t po = (size_t)b * N * kXcaC * es;
      pfb_conv_params p{};
      p.src[0].ptr = reinterpret_cast<const char*>(v_ln) + po; p.src[0].channels = kXcaC; p.src[0].stride = kXcaC;
      p.nsrc = 1;
      p.B = 1; p.H = c->H; p.W = c->W; p.KH = 1; p.KW = 1;
      p.Cout = kXcaC; p.Cout_pad = kXcaC; p.weight = wf + (size_t)b * kXcaC * kXcaC * es; p.bias = nullptr;
      p.epilogue = PFB_EPI_AXPY; p.scale = 1.f;
      p.out = reinterpret_cast<char*>(x1) + po; p.out_stride = kXcaC; p.out_offset = 0;
      p.aux_h = reinterpret_cast<char*>(add) + po; p.hidden = kXcaC;
      p.dtype = c->dtype; p.impl = 1;
      PFB_TRY(pfb_conv2d(&p, st));
    }
  }
  // x2 = x1 + gamma3 * LPI(LN3(x1)): LN3's affine and the group norm's are applied, not folded (the convolutions are zero padded)
  PFB_TRY(pfb_layernorm(x1, kXcaC, 0, t, kXcaC, 0, w.ln3_weight, w.ln3_bias, P, kXcaC, w.ln_eps, c->dtype, st));
  PFB_TRY(pfb_depthwise_conv3x3_ex(t, kXcaC, 0, u, kXcaC, 0, w.dw1_weight, w.dw1_bias, nullptr, 0, 0, c->B, c->H, c->W, kXcaC, 0, c->dtype, st));
  PFB_TRY(pfb_group_norm_act(u, u, nullptr, x.at(x.pl.off_gn), nullptr, w.gn_weight, w.gn_bias, c->B, c->H, c->W, kXcaC, kXcaC / 8, w.gn_eps,
                             0, c->dtype, st));
  PFB_TRY(pfb_depthwise_conv3x3_ex(u, kXcaC, 0, t, kXcaC, 0, w.dw2_weight, w.dw2_bias, x1, kXcaC, 0, c->B, c->H, c->W, kXcaC, 1, c->dtype, st));
  // out = x2 + gamma2 * fc2(gelu(fc1(LN2(x2))))
  PFB_TRY(pfb_layernorm(t, kXcaC, 0, u, kXcaC, 0, nullptr, nullptr, P, kXcaC, w.ln_eps, c->dtype, st));
  PFB_TRY(conv1x1s(x, w.fc1, c->B, c->H, c->W, u, kXcaC, 0, PFB_EPI_GELU, x1, kXcaC, 0));
  return conv1x1s(x, w.fc2, c->B, c->H, c->W, x1, kXcaC, 0, PFB_EPI_AXPY, out, out_stride, out_offset, t, kXcaC);
}

static int positional(const Xs& x, const pfb_xcit_block& w, size_t off) {
  PFB_CHECK_ARG(w.pos_proj.Cin == 64 && w.pos_proj.Cout == kXcaC, "ccmr: pos_embeder.token_projection must be 64 -> 128");
  return conv1x1s(x, w.pos_proj, 1, x.c->H, x.c->W, x.at(x.pl.off_feat), 64, 0, PFB_EPI_LINEAR, x.at(off), kXcaC, 0);
}

int ccmr_scale_setup(const pfb_raft_cfg* c, const pfb_ccmr_weights* w, const void* inp, void* gc_out, bool aggregator, char* base,
                     cudaStream_t s) {
  Xs x{c, ccmr_plan(c), base, s};
  const int N = c->H * c->W;
  PFB_TRY(pfb_fourier_features(x.at(x.pl.off_feat), c->H, c->W, c->dtype, (pfb_stream)s));
  PFB_TRY(positional(x, w->context, x.pl.off_pos_c));
  // global_context = XCiT(inp): x = inp + pos, one self-attention block (v from the same LN1 output as q and k)
  PFB_TRY(xcit_residual(inp, kXcaC, x.at(x.pl.off_pos_c), nullptr, x.at(x.pl.off_x0), c->B, N, c->dtype, s));
  PFB_TRY(xcit_prepare(x, w->context));
  void* gc = gc_out ? gc_out : x.at(x.pl.off_gc);
  PFB_TRY(xcit_apply(x, w->context, x.at(x.pl.off_ln), gc, kXcaC, 0));
  if (!aggregator) return PFB_OK;
  // the aggregator's residual stream global_context + pos and its attention, constant over the scale's iterations
  PFB_TRY(positional(x, w->aggregator, x.pl.off_pos_a));
  PFB_TRY(xcit_residual(gc, kXcaC, x.at(x.pl.off_pos_a), nullptr, x.at(x.pl.off_x0), c->B, N, c->dtype, s));
  return xcit_prepare(x, w->aggregator);
}

int ccmr_aggregate(const pfb_raft_cfg* c, const pfb_ccmr_weights* w, void* motion, int motion_stride, char* base, cudaStream_t s) {
  Xs x{c, ccmr_plan(c), base, s};
  const size_t P = (size_t)c->B * c->H * c->W;
  void* ln = x.at(x.pl.off_ln);
  PFB_TRY(pfb_layernorm(motion, motion_stride, 0, ln, kXcaC, 0, nullptr, nullptr, P, kXcaC, w->aggregator.ln_eps, c->dtype, (pfb_stream)s));
  return xcit_apply(x, w->aggregator, ln, motion, motion_stride, kXcaC);
}

int ccmr_output(const pfb_raft_cfg* c, const float* coords, const void* mask, float* flow_up, float* flow_small, int upflow2, char* base,
                cudaStream_t s) {
  const pfb_stream st = (pfb_stream)s;
  if (upflow2) {
    float* up = reinterpret_cast<float*>(base + ccmr_plan(c).off_up);
    PFB_TRY(pfb_convex_upsample2x(coords, mask, up, 0, c->B, c->H, c->W, 2 * c->H, 2 * c->W, 0, 0, c->dtype, st));
    PFB_TRY(pfb_upflow2(up, flow_up, c->B, 2 * c->H, 2 * c->W, c->out_h, c->out_w, c->pad_top, c->pad_left, st));
  } else {
    PFB_TRY(pfb_convex_upsample2x(coords, mask, flow_up, 0, c->B, c->H, c->W, c->out_h, c->out_w, c->pad_top, c->pad_left, c->dtype, st));
  }
  if (!flow_small) return PFB_OK;
  return pfb_downflow(flow_up, flow_small, c->B, c->out_h, c->out_w, c->out_h / 16, c->out_w / 16, st);
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_fourier_features(void* out, int H, int W, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(out, "fourier_features: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && H > 0 && W > 0, "fourier_features: bad arguments %dx%d", H, W);
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, { fourier_features_kernel<T><<<grid_for((size_t)H * W * 64), 256, 0, s>>>((T*)out, H, W); });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API size_t pfb_xca_stats_workspace_bytes(int B, int N) {
  if (B <= 0 || N <= 0) return 0;
  return (size_t)B * ceil_div_sz((size_t)N, kXcaChunk) * kXcaStats * sizeof(float);
}

extern "C" PFB_API int pfb_xca_stats(const void* qk, int qk_stride, int q_offset, int k_offset, int B, int N, float* stats, void* workspace,
                                     pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(qk && stats && workspace, "xca_stats: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && B <= 65535 && N > 0, "xca_stats: bad shape B=%d N=%d", B, N);
  PFB_CHECK_ARG(q_offset >= 0 && k_offset >= 0 && qk_stride >= q_offset + kXcaC && qk_stride >= k_offset + kXcaC,
                "xca_stats: q / k columns (%d, %d, 128 each) outside the row of %d", q_offset, k_offset, qk_stride);
  cudaStream_t s = as_stream(stream);
  const int chunks = ceil_div(N, kXcaChunk);
  float* part = reinterpret_cast<float*>(workspace);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    xca_stats_kernel<T><<<dim3(chunks, B), 256, 0, s>>>((const T*)qk, qk_stride, q_offset, k_offset, N, chunks, part);
  });
  PFB_LAUNCH_CHECK();
  xca_combine_kernel<<<dim3(ceil_div(kXcaStats, 256), B), 256, 0, s>>>(part, chunks, stats);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_xca_fold(const float* stats, const float* temperature, const float* v_w, const float* v_b, const float* proj_w,
                                    const float* proj_b, void* w_out, void* w_out_k, float* bias_out, int B, pfb_dtype dtype,
                                    pfb_stream stream) {
  PFB_CHECK_ARG(stats && temperature && v_w && v_b && proj_w && proj_b && w_out && bias_out, "xca_fold: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype) && B > 0 && B <= 65535, "xca_fold: bad arguments (B=%d)", B);
  cudaStream_t s = as_stream(stream);
  static std::atomic<unsigned long long> attr_done{0};
  int dev = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  if (!(attr_done.load(std::memory_order_acquire) & (1ull << (dev & 63)))) {
    PFB_CUDA(cudaFuncSetAttribute(xca_fold_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFoldSmem));
    PFB_CUDA(cudaFuncSetAttribute(xca_fold_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFoldSmem));
    PFB_CUDA(cudaFuncSetAttribute(xca_fold_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFoldSmem));
    attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
  }
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    xca_fold_kernel<T><<<dim3(B, kXcaC / 16), 256, kFoldSmem, s>>>(stats, temperature, v_w, v_b, proj_w, proj_b, (T*)w_out, (T*)w_out_k,
                                                                    bias_out);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_upflow2(const float* flow, float* out, int B, int H, int W, int out_h, int out_w, int pad_top, int pad_left,
                                   pfb_stream stream) {
  PFB_CHECK_ARG(flow && out, "upflow2: null pointer");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0 && pad_top >= 0 && pad_left >= 0 && out_h + pad_top <= 2 * H &&
                    out_w + pad_left <= 2 * W,
                "upflow2: output window %dx%d+(%d,%d) outside %dx%d", out_h, out_w, pad_top, pad_left, 2 * H, 2 * W);
  cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_UPSAMPLE, s);
  upflow2_kernel<<<grid_for((size_t)B * out_h * out_w), 256, 0, s>>>(flow, out, B, H, W, out_h, out_w, pad_top, pad_left);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
