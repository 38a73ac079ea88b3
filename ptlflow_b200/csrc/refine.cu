// Host-side orchestration of the refinement loop: lookup -> motion encoder -> GRU -> heads,
// `iters` times, then the upsample.  Mirrors the data flow of
//   ptlflow/models/raft/raft.py:170-192 and ptlflow/models/raft/update.py:115-153
// but every stage is one launch of this library's kernels on the caller's stream (so the whole
// loop can be captured in a CUDA graph by the host), no torch.cat / permute copies exist, and
// the mask head + upsample run once (eval returns only the last prediction, raft.py:192).
#include <initializer_list>

#include <stdlib.h>

#include "refine.cuh"

#define PFB_TRY(expr)        \
  do {                       \
    int rc__ = (expr);       \
    if (rc__ != PFB_OK) return rc__; \
  } while (0)

namespace pfb {

struct Workspace {
  // element strides (channels per pixel) and byte offsets inside the caller's workspace
  int planes, corr_stride;
  size_t off_corr, off_cor1, off_corflo, off_flo1, off_motion, off_z, off_rh, off_fh, off_mh, off_mask, off_flow;
  size_t off_taps;          // flow head conv2 per-tap products [P][32] fp32 (tensor-core path)
  size_t off_vbuf, off_vT;  // gma: to_v(motion) [P][heads*128] and its per-sample transpose [B][heads*128][n_pad]
  size_t off_agg;           // gma, heads > 1: the concatenated per-head attn @ v [P][heads*128] (input of Aggregate.project)
  size_t off_flags;         // on-the-fly tensor-core lookup: one flag per query (queries recomputed by the SIMT pass)
  size_t off_ctx[4];        // iteration-invariant context terms of the GRU gates: zr1 [P][2hd], q1 [P][hd], zr2, q2 (tensor path)
  int n_pad;
  size_t total;
  int c_cor1, c_corflo, c_cor2, c_flo1, c_flo2, c_motion, c_fh;
};

static int heads_of(const pfb_raft_cfg* c) { return c->num_heads > 0 ? c->num_heads : 1; }
// channels of the convex-upsample mask: 9 taps x 8 x 8 (raft, gma), 9 taps x 2 x 2 (ms_raft_plus, variant 5; ccmr, variant 6)
static int mask_channels(const pfb_raft_cfg* c) { return c->variant == 5 || c->variant == 6 ? 36 : 576; }

static Workspace plan(const pfb_raft_cfg* c) {
  Workspace w{};
  const size_t vdim = (size_t)heads_of(c) * 128;
  const size_t P = (size_t)c->B * c->H * c->W;
  const size_t es = dtype_size(c->dtype);
  const int K = 2 * c->corr_radius + 1;
  w.planes = c->corr_levels * K * K;
  // 16-byte aligned rows for the tensor-core path (the TMA unit zero-fills a partial last 64-channel K chunk itself)
  w.corr_stride = (c->dtype == PFB_F32) ? w.planes : (int)align_up(w.planes, 8);
  if (c->variant == 0 || c->variant == 2 || c->variant == 5 || c->variant == 6) {
    w.c_cor1 = 256; w.c_cor2 = 192; w.c_flo1 = 128; w.c_flo2 = 64; w.c_fh = 256;
    // gma and ccmr keep [motion | motion_global] side by side so the GRU still sees three sources (update.py:150-151)
    w.c_motion = c->variant == 2 || c->variant == 6 ? 256 : 128;
  } else {
    w.c_cor1 = 0; w.c_cor2 = 96; w.c_flo1 = 64; w.c_flo2 = 32; w.c_motion = 82; w.c_fh = 128;
  }
  w.c_corflo = w.c_cor2 + w.c_flo2;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  w.off_corr = take(P * w.corr_stride * es);
  w.off_cor1 = take(P * (size_t)w.c_cor1 * es);
  w.off_corflo = take(P * (size_t)w.c_corflo * es);
  w.off_flo1 = take(P * (size_t)w.c_flo1 * es);
  w.off_motion = take(P * (size_t)w.c_motion * es);
  w.off_z = take(P * (size_t)c->hidden_dim * es);
  w.off_rh = take(P * (size_t)c->hidden_dim * es);
  w.off_fh = take(P * (size_t)w.c_fh * es);
  w.off_mh = take(c->variant != 1 ? P * 256 * es : 0);
  w.off_mask = take(c->variant != 1 ? P * (size_t)mask_channels(c) * es : 0);
  w.off_flow = take(P * 2 * sizeof(float));
  w.off_taps = take(c->variant != 1 ? P * 32 * sizeof(float) : 0);
  w.n_pad = (int)align_up((size_t)c->H * c->W, 64);
  w.off_vbuf = take(c->variant == 2 ? P * vdim * es : 0);
  w.off_vT = take(c->variant == 2 ? (size_t)c->B * vdim * w.n_pad * es : 0);
  w.off_agg = take(c->variant == 2 && vdim > 128 ? P * vdim * es : 0);
  w.off_flags = take(c->alternate_corr ? P : 0);
  for (int i = 0; i < 4; ++i)
    w.off_ctx[i] = take((c->variant != 1 && c->dtype != PFB_F32) ? P * (size_t)((i & 1) ? c->hidden_dim : 2 * c->hidden_dim) * es : 0);
  w.total = off;
  return w;
}

// variant 5 (ms_raft_plus) only through the pfb_msraft_* entry points, 6 (ccmr) only through the pfb_ccmr_* ones, 0..2 only through
// the pfb_raft_* ones
static int check_cfg(const pfb_raft_cfg* c, bool msraft = false, bool ccmr = false) {
  PFB_CHECK_ARG(c, "raft: null cfg");
  if (ccmr) PFB_CHECK_ARG(c->variant == 6, "ccmr: variant=%d (the ccmr loop is variant 6)", c->variant);
  else if (msraft) PFB_CHECK_ARG(c->variant == 5, "msraft: variant=%d (the ms_raft_plus loop is variant 5)", c->variant);
  else PFB_CHECK_ARG(c->variant >= 0 && c->variant <= 2, "raft: variant=%d", c->variant);
  PFB_CHECK_ARG(dtype_ok(c->dtype), "raft: bad dtype");
  PFB_CHECK_ARG(c->B > 0 && c->H > 0 && c->W > 0, "raft: bad grid %dx%dx%d", c->B, c->H, c->W);
  PFB_CHECK_ARG(c->corr_levels >= 1 && c->corr_levels <= PFB_MAX_LEVELS && c->corr_radius >= 0 && c->corr_radius <= 15,
                "raft: corr_levels=%d corr_radius=%d", c->corr_levels, c->corr_radius);
  PFB_CHECK_ARG((c->H >> (c->corr_levels - 1)) >= 1 && (c->W >> (c->corr_levels - 1)) >= 1,
                "raft: %dx%d grid too small for %d levels", c->H, c->W, c->corr_levels);
  PFB_CHECK_ARG(c->hidden_dim > 0 && c->context_dim > 0 && c->iters >= 0, "raft: bad dims");
  PFB_CHECK_ARG(c->num_heads >= 0 && c->num_heads <= 64 && (c->variant == 2 || heads_of(c) == 1), "raft: num_heads=%d", c->num_heads);
  PFB_CHECK_ARG(c->volume_layout == 0 || (c->volume_layout == 1 && c->dtype != PFB_F32 && !c->alternate_corr && c->corr_levels <= 4),
                "raft: volume_layout=%d needs f16/bf16, a materialised pyramid and <= 4 levels", c->volume_layout);
  if (c->variant != 1) PFB_CHECK_ARG(c->hidden_dim == 128 && c->context_dim == 128, "raft/gma: the update block expects hidden=context=128");
  else PFB_CHECK_ARG(c->hidden_dim == 96 && c->context_dim == 64, "raft_small: SmallUpdateBlock expects hidden=96 context=64");
  return PFB_OK;
}

struct Ctx {
  const pfb_raft_cfg* c;
  const pfb_raft_weights* w;
  const pfb_raft_buffers* b;
  Workspace ws;
  char* base;
  cudaStream_t s;
  float corr_scale = 0.f;  // on-the-fly lookup scale (0: 1/sqrt(feat_dim))
  const pfb_ccmr_weights* ccmr = nullptr;  // variant 6: the XCiT blocks of the scale, and their part of the workspace
  char* ccmr_base = nullptr;
  // flow branch of the motion encoder on a second stream (fork_flow_branch): null when not forked
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  void* at(size_t off) const { return base + off; }
};

static pfb_conv_src src_of(const void* ptr, int channels, int stride, int offset = 0, int is_f32 = 0) {
  pfb_conv_src s;
  s.ptr = ptr; s.channels = channels; s.stride = stride; s.offset = offset; s.is_f32 = is_f32;
  return s;
}

static int run_conv(const Ctx& x, int layer, std::initializer_list<pfb_conv_src> srcs, int epi, void* out,
                    int out_stride, int out_offset, float scale = 1.f, const void* addend = nullptr, int addend_stride = 0) {
  const pfb_layer& L = x.w->layers[layer];
  PFB_CHECK_ARG(L.weight, "raft: layer %d has no packed weight", layer);
  pfb_conv_params p{};
  int i = 0, cin = 0;
  for (const auto& s : srcs) { p.src[i++] = s; cin += s.channels; }
  p.nsrc = i;
  // the lookup buffer may be wider than the layer's real Cin (zero pad columns <-> zero weight rows)
  PFB_CHECK_ARG(cin == L.Cin, "raft: layer %d expects Cin=%d, sources provide %d", layer, L.Cin, cin);
  p.B = x.c->B; p.H = x.c->H; p.W = x.c->W;
  p.KH = L.KH; p.KW = L.KW; p.Cout = L.Cout; p.Cout_pad = L.Cout_pad;
  p.weight = L.weight; p.bias = L.bias;
  p.epilogue = epi; p.scale = scale;
  p.out = out; p.out_stride = out_stride; p.out_offset = out_offset;
  p.aux_h = x.b->net; p.aux_z = x.at(x.ws.off_z); p.hidden = x.c->hidden_dim;
  p.coords = x.b->coords; p.flow = reinterpret_cast<const float*>(x.at(x.ws.off_flow));
  p.dtype = x.c->dtype; p.impl = x.c->impl;
  p.weight_k = L.weight_k; p.Cin_pad = L.Cin_pad; p.Cout_pad_k = L.Cout_pad_k;
  p.addend = addend; p.addend_stride = addend_stride;
  return pfb_conv2d(&p, (pfb_stream)x.s);
}

// round-2 restructurings of the tensor-core path; PFB_GRU_CTX_SPLIT=0 / PFB_MERGE_C2F2=0 fall back to the plain layers
static bool tensor_path(const Ctx& x) { return x.c->variant != 1 && x.c->dtype != PFB_F32 && x.c->impl != 1; }
static bool ctx_split_active(const Ctx& x) {
  static const int env = getenv("PFB_GRU_CTX_SPLIT") ? atoi(getenv("PFB_GRU_CTX_SPLIT")) : 1;
  return env && tensor_path(x) && x.w->layers[PFB_L_GRUX_ZR1].weight_k && x.w->layers[PFB_L_CTX_ZR1].weight_k;
}
static bool merged_c2f2_active(const Ctx& x) {
  // measured (launch list r02b): 70.5 us merged vs 46.3 + 23.8 us separate -- the zero blocks cost what the better shape saves,
  // so the merged layer is opt-in
  static const int env = getenv("PFB_MERGE_C2F2") ? atoi(getenv("PFB_MERGE_C2F2")) : 0;
  return env && tensor_path(x) && x.w->layers[PFB_L_CONVC2F2].weight_k;
}
// The motion encoder has two independent branches: lookup -> convc1 -> convc2 (correlation) and convf1 -> convf2 (flow); both
// start from the previous iteration's coordinates and meet in `conv`.  cfg.fork_flow puts the flow branch on a second stream
// of this host thread (fork / join with events, which a CUDA-graph capture turns into parallel branches of the graph), so that
// the SIMT lookup can share the SMs with the two small tensor-core layers (+0.3 ... 2 % per step, DESIGN.md section 4).
static bool fork_flow_active(const Ctx& x) { return x.c->fork_flow && tensor_path(x) && !merged_c2f2_active(x); }
static int fork_flow_setup(Ctx& x) {
  if (!fork_flow_active(x)) return PFB_OK;
  // one side stream + event pair per (host thread, device): forwards of different host threads run concurrently
  struct Lane {
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  };
  constexpr int kMaxDev = 64;
  thread_local Lane lanes[kMaxDev];
  int dev = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= kMaxDev) return PFB_OK;  // no fork on exotic device numbers: everything stays on the caller's stream
  Lane& l = lanes[dev];
  if (!l.side) {
    PFB_CUDA(cudaStreamCreateWithFlags(&l.side, cudaStreamNonBlocking));
    PFB_CUDA(cudaEventCreateWithFlags(&l.ev_fork, cudaEventDisableTiming));
    PFB_CUDA(cudaEventCreateWithFlags(&l.ev_join, cudaEventDisableTiming));
  }
  x.side = l.side; x.ev_fork = l.ev_fork; x.ev_join = l.ev_join;
  return PFB_OK;
}

// conv_inp(inp) + bias for the four GRU convolutions: once per forward (inp does not change over the iterations)
static int run_context_terms(const Ctx& x) {
  if (!ctx_split_active(x)) return PFB_OK;
  const int hd = x.c->hidden_dim, cd = x.c->context_dim;
  const int layers[4] = {PFB_L_CTX_ZR1, PFB_L_CTX_Q1, PFB_L_CTX_ZR2, PFB_L_CTX_Q2};
  for (int i = 0; i < 4; ++i) {
    const int n = (i & 1) ? hd : 2 * hd;
    PFB_TRY(run_conv(x, layers[i], {src_of(x.b->inp, cd, cd)}, PFB_EPI_LINEAR, x.at(x.ws.off_ctx[i]), n, 0));
  }
  return PFB_OK;
}

int raft_lookup(const pfb_raft_cfg* c, void* const* pyramid, const void* fmap1, const float* coords, void* out, int out_stride,
                void* flags, cudaStream_t s, float scale) {
  if (c->alternate_corr) {
    static const int env_tc = getenv("PFB_ONTHEFLY_TC") ? atoi(getenv("PFB_ONTHEFLY_TC")) : 1;
    if (env_tc && c->impl != 1 && corr_onthefly_umma_supported(c->B, c->H, c->W, c->feat_dim, c->corr_levels, c->corr_radius, c->dtype, out_stride))
      return pfb_corr_lookup_onthefly_tc_ex(fmap1, pyramid, coords, out, flags, c->B, c->H, c->W,
                                            c->feat_dim, c->corr_levels, c->corr_radius, scale, c->dtype, out_stride, (pfb_stream)s);
  }
  if (c->alternate_corr)
    return pfb_corr_lookup_onthefly_ex(fmap1, pyramid, coords, out, c->B, c->H, c->W,
                                       c->feat_dim, c->corr_levels, c->corr_radius, scale, c->dtype, c->dtype, 0,
                                       out_stride, (pfb_stream)s);
  if (c->volume_layout == 1)
    return pfb_corr_lookup_tiled(pyramid, coords, out, c->B, c->H, c->W, c->H, c->W, c->corr_levels,
                                 c->corr_radius, c->dtype, out_stride, (pfb_stream)s);
  return pfb_corr_lookup(pyramid, coords, out, c->B, c->H, c->W, c->corr_levels,
                         c->corr_radius, c->dtype, c->dtype, 0, out_stride, (pfb_stream)s);
}

static int lookup(const Ctx& x) {
  return raft_lookup(x.c, x.b->pyramid, x.b->fmap1, x.b->coords, x.at(x.ws.off_corr), x.ws.corr_stride, x.at(x.ws.off_flags), x.s,
                     x.corr_scale);
}

int gma_aggregate(const pfb_raft_cfg* c, const pfb_layer& agg_v, const pfb_layer& agg_proj, const void* attention_ptr, float gamma,
                  void* motion, int motion_stride, int motion_offset, int out_offset, void* vbuf_ptr, void* vT_ptr, void* agg_ptr, int n_pad,
                  cudaStream_t s) {
  PFB_CHECK_ARG(attention_ptr, "gma: null attention");
  const int N = c->H * c->W, heads = heads_of(c), vdim = heads * 128;
  const size_t es = dtype_size(c->dtype);
  const char* attention = reinterpret_cast<const char*>(attention_ptr);
  char* vbuf = reinterpret_cast<char*>(vbuf_ptr);
  char* vT = reinterpret_cast<char*>(vT_ptr);
  // one head: attn @ v goes straight into the AXPY epilogue.  Several heads (gma_utils.py:101-111): every head's attn @ v
  // lands in its 128 columns of `agg`, then project (heads*128 -> 128) carries the AXPY epilogue.
  char* agg = heads > 1 ? reinterpret_cast<char*>(agg_ptr) : nullptr;
  PFB_CHECK_ARG(heads == 1 || (agg_proj.weight && agg_proj.Cin == vdim),
                "gma: num_heads=%d needs the Aggregate.project layer (%d -> 128)", heads, vdim);
  PFB_CHECK_ARG(agg_v.weight && agg_v.Cin == 128, "gma: Aggregate.to_v layer missing");
  {  // v = to_v(motion)
    pfb_conv_params p{};
    p.src[0] = src_of(motion, 128, motion_stride, motion_offset);
    p.nsrc = 1;
    p.B = c->B; p.H = c->H; p.W = c->W; p.KH = agg_v.KH; p.KW = agg_v.KW;
    p.Cout = agg_v.Cout; p.Cout_pad = agg_v.Cout_pad;
    p.weight = agg_v.weight; p.bias = agg_v.bias;
    p.epilogue = PFB_EPI_LINEAR; p.scale = 1.f;
    p.out = vbuf; p.out_stride = vdim; p.out_offset = 0;
    p.hidden = c->hidden_dim;
    p.dtype = c->dtype; p.impl = c->impl;
    p.weight_k = agg_v.weight_k; p.Cin_pad = agg_v.Cin_pad; p.Cout_pad_k = agg_v.Cout_pad_k;
    PFB_TRY(pfb_conv2d(&p, (pfb_stream)s));
  }
  const bool tensor_path = c->dtype != PFB_F32 && c->impl != 1 && (N % 8) == 0;
  if (tensor_path) PFB_TRY(pfb_transpose_pm(vbuf, vT, c->B, N, vdim, n_pad, c->dtype, (pfb_stream)s));
  static const int env_batched = getenv("PFB_GMA_BATCHED") ? atoi(getenv("PFB_GMA_BATCHED")) : 1;
  // "1x1 convolution" of head h over sample b (b < 0: all samples in one launch): pixels = queries, input channels = the N
  // attention columns, weights = the sample's v (SIMT layout [N][vdim], columns h*128...) / v^T (K-major [vdim][n_pad], rows
  // h*128...).  The attention is head-major, so every operand is affine in the pixel index.
  auto attn_v = [&](int h, int b) -> int {
    const int b0 = b < 0 ? 0 : b;
    pfb_conv_params p{};
    p.src[0] = src_of(attention + ((size_t)h * c->B + b0) * N * N * es, N, N);
    p.nsrc = 1;
    p.B = b < 0 ? c->B : 1; p.H = c->H; p.W = c->W; p.KH = 1; p.KW = 1;
    p.Cout = 128; p.Cout_pad = vdim;
    p.weight = vbuf + ((size_t)b0 * N * vdim + (size_t)h * 128) * es;
    p.bias = nullptr;
    if (heads == 1) {
      char* mrow = reinterpret_cast<char*>(motion) + (size_t)b0 * N * motion_stride * es;
      p.epilogue = PFB_EPI_AXPY; p.scale = gamma;
      p.out = mrow; p.out_stride = motion_stride; p.out_offset = out_offset;
      p.aux_h = mrow + (size_t)motion_offset * es; p.hidden = motion_stride;
    } else {
      p.epilogue = PFB_EPI_LINEAR; p.scale = 1.f;
      p.out = agg + (size_t)b0 * N * vdim * es; p.out_stride = vdim; p.out_offset = h * 128;
    }
    p.dtype = c->dtype; p.impl = c->impl;
    if (tensor_path) {
      p.weight_k = vT + ((size_t)b0 * vdim + (size_t)h * 128) * n_pad * es; p.Cin_pad = n_pad; p.Cout_pad_k = 128;
    }
    if (b < 0) {
      // ONE launch for all samples: per-sample weights = that sample's v^T (rows b * vdim + h * 128 ...).  B x 55 row tiles
      // fill the machine; one launch per sample left only 55 row tiles, a fraction of the machine.
      p.impl = 2;
      p.w_rows_per_sample = vdim;
    }
    return pfb_conv2d(&p, (pfb_stream)s);
  };
  for (int h = 0; h < heads; ++h) {
    if (tensor_path && env_batched) PFB_TRY(attn_v(h, -1));
    else for (int b = 0; b < c->B; ++b) PFB_TRY(attn_v(h, b));
  }
  if (heads > 1) {  // motion_global = motion + gamma * project(out)   gma_utils.py:108-111
    const pfb_layer& L = agg_proj;
    pfb_conv_params p{};
    p.src[0] = src_of(agg, vdim, vdim);
    p.nsrc = 1;
    p.B = c->B; p.H = c->H; p.W = c->W; p.KH = 1; p.KW = 1;
    p.Cout = L.Cout; p.Cout_pad = L.Cout_pad;
    p.weight = L.weight; p.bias = nullptr;
    p.epilogue = PFB_EPI_AXPY; p.scale = gamma;
    p.out = motion; p.out_stride = motion_stride; p.out_offset = out_offset;
    p.aux_h = reinterpret_cast<char*>(motion) + (size_t)motion_offset * es; p.hidden = motion_stride;
    p.dtype = c->dtype; p.impl = c->impl;
    p.weight_k = L.weight_k; p.Cin_pad = L.Cin_pad; p.Cout_pad_k = L.Cout_pad_k;
    PFB_TRY(pfb_conv2d(&p, (pfb_stream)s));
  }
  return PFB_OK;
}

// One BasicUpdateBlock / SmallUpdateBlock evaluation + coords update.  update.py:122-153
static int update_iter(const Ctx& x, const void* corr_ext, void* mask_out) {
  const pfb_raft_cfg* c = x.c;
  const Workspace& ws = x.ws;
  const int hd = c->hidden_dim, cd = c->context_dim;
  const void* corr = corr_ext ? corr_ext : x.at(ws.off_corr);
  const int corr_stride = corr_ext ? ws.planes : ws.corr_stride;
  void* corflo = x.at(ws.off_corflo);
  void* flo1 = x.at(ws.off_flo1);
  void* motion = x.at(ws.off_motion);
  void* rh = x.at(ws.off_rh);
  void* fh = x.at(ws.off_fh);
  float* flow = reinterpret_cast<float*>(x.at(ws.off_flow));

  // ---- motion encoder (update.py:76-112) ----
  const bool merged_c2f2 = merged_c2f2_active(x);
  Ctx xf = x;  // the flow branch's launches: the side stream when forked (the fork itself is in the caller, before the lookup)
  if (x.side) xf.s = x.side;
  if (c->variant != 1) {
    void* cor1 = x.at(ws.off_cor1);
    PFB_TRY(run_conv(x, PFB_L_CONVC1, {src_of(corr, ws.planes, corr_stride)}, PFB_EPI_RELU, cor1, ws.c_cor1, 0));
    if (!merged_c2f2) PFB_TRY(run_conv(x, PFB_L_CONVC2, {src_of(cor1, ws.c_cor1, ws.c_cor1)}, PFB_EPI_RELU, corflo, ws.c_corflo, 0));
  } else {
    PFB_TRY(run_conv(x, PFB_L_CONVC1, {src_of(corr, ws.planes, corr_stride)}, PFB_EPI_RELU, corflo, ws.c_corflo, 0));
  }
  {
    const pfb_layer& LF = x.w->layers[PFB_L_CONVF1];
    static const int env_fc = getenv("PFB_FLOW_CONV_UMMA") ? atoi(getenv("PFB_FLOW_CONV_UMMA")) : 1;
    if (env_fc && LF.weight_k && LF.KH == 7 && LF.KW == 7 && LF.Cin == 2 && LF.Cout == 128 && c->dtype != PFB_F32 && c->impl != 1)
      PFB_TRY(pfb_flow_conv7x7(flow, LF.weight_k, LF.bias, flo1, ws.c_flo1, 0, c->B, c->H, c->W, c->dtype, (pfb_stream)xf.s));
    else
      PFB_TRY(run_conv(xf, PFB_L_CONVF1, {src_of(flow, 2, 2, 0, 1)}, PFB_EPI_RELU, flo1, ws.c_flo1, 0));
  }
  if (merged_c2f2)  // convc2 | convf2 as one block-diagonal layer: [cor1 (256) | flo1 (128)] -> [cor (192) | flo (64)]
    PFB_TRY(run_conv(x, PFB_L_CONVC2F2, {src_of(x.at(ws.off_cor1), ws.c_cor1, ws.c_cor1), src_of(flo1, ws.c_flo1, ws.c_flo1)}, PFB_EPI_RELU,
                     corflo, ws.c_corflo, 0));
  else
    PFB_TRY(run_conv(xf, PFB_L_CONVF2, {src_of(flo1, ws.c_flo1, ws.c_flo1)}, PFB_EPI_RELU, corflo, ws.c_corflo, ws.c_cor2));
  if (x.side) {  // join: `conv` reads both branches
    PFB_CUDA(cudaEventRecord(x.ev_join, x.side));
    PFB_CUDA(cudaStreamWaitEvent(x.s, x.ev_join, 0));
  }
  PFB_TRY(run_conv(x, PFB_L_CONV, {src_of(corflo, ws.c_corflo, ws.c_corflo)}, PFB_EPI_RELU_APPEND_FLOW, motion, ws.c_motion, 0));

  // ---- gma: motion_global = motion + gamma * (attention @ to_v(motion))   gma_utils.py:101-113, gma/update.py:149 ----
  if (c->variant == 2)
    PFB_TRY(gma_aggregate(c, x.w->layers[PFB_L_AGG_V], x.w->layers[PFB_L_AGG_PROJ], x.b->attention, x.b->agg_gamma, motion, ws.c_motion, 0,
                          128, x.at(ws.off_vbuf), x.at(ws.off_vT), x.at(ws.off_agg), ws.n_pad, x.s));
  // ---- ccmr: motion_global = aggregator(global_context, motion)   ccmr/update.py:156-161 ----
  if (c->variant == 6) PFB_TRY(ccmr_aggregate(c, x.ccmr, motion, ws.c_motion, x.ccmr_base, x.s));

  // ---- GRU (update.py:24-32 ConvGRU, :58-73 SepConvGRU); x = [inp, motion (, motion_global)] ----
  const int halves = (c->variant != 1) ? 2 : 1;
  const bool split = ctx_split_active(x);
  for (int h = 0; h < halves; ++h) {
    if (split) {
      // conv([h | inp | motion]) = conv_inp(inp) + bias (once per forward, run_context_terms) + conv_rest([h | motion]) (here)
      const int lzr = h == 0 ? PFB_L_GRUX_ZR1 : PFB_L_GRUX_ZR2, lq = h == 0 ? PFB_L_GRUX_Q1 : PFB_L_GRUX_Q2;
      PFB_TRY(run_conv(x, lzr, {src_of(x.b->net, hd, hd), src_of(motion, ws.c_motion, ws.c_motion)}, PFB_EPI_GRU_ZR, rh, hd, 0, 1.f,
                       x.at(ws.off_ctx[2 * h]), 2 * hd));
      PFB_TRY(run_conv(x, lq, {src_of(rh, hd, hd), src_of(motion, ws.c_motion, ws.c_motion)}, PFB_EPI_GRU_Q, x.b->net, hd, 0, 1.f,
                       x.at(ws.off_ctx[2 * h + 1]), hd));
      continue;
    }
    const int lzr = h == 0 ? PFB_L_GRU_ZR1 : PFB_L_GRU_ZR2, lq = h == 0 ? PFB_L_GRU_Q1 : PFB_L_GRU_Q2;
    PFB_TRY(run_conv(x, lzr, {src_of(x.b->net, hd, hd), src_of(x.b->inp, cd, cd), src_of(motion, ws.c_motion, ws.c_motion)},
                     PFB_EPI_GRU_ZR, rh, hd, 0));
    PFB_TRY(run_conv(x, lq, {src_of(rh, hd, hd), src_of(x.b->inp, cd, cd), src_of(motion, ws.c_motion, ws.c_motion)},
                     PFB_EPI_GRU_Q, x.b->net, hd, 0));
  }

  // ---- heads (update.py:6-14, :138-152) ----
  const bool fork_mask = x.side && mask_out && c->variant != 1;
  if (fork_mask) {  // last iteration: the mask head beside the flow head (both read the final hidden state)
    PFB_CUDA(cudaEventRecord(x.ev_fork, x.s));
    PFB_CUDA(cudaStreamWaitEvent(x.side, x.ev_fork, 0));
    void* mh = x.at(ws.off_mh);
    PFB_TRY(run_conv(xf, PFB_L_MASK1, {src_of(x.b->net, hd, hd)}, PFB_EPI_RELU, mh, 256, 0));
    PFB_TRY(run_conv(xf, PFB_L_MASK2, {src_of(mh, 256, 256)}, PFB_EPI_LINEAR, mask_out, mask_channels(c), 0, 0.25f));
    PFB_CUDA(cudaEventRecord(x.ev_join, x.side));
  }
  PFB_TRY(run_conv(x, PFB_L_FLOW1, {src_of(x.b->net, hd, hd)}, PFB_EPI_RELU, fh, ws.c_fh, 0));
  const pfb_layer& LT = x.w->layers[PFB_L_FLOW2T];
  if (c->variant != 1 && c->dtype != PFB_F32 && c->impl != 1 && LT.weight_k) {
    // tensor-core form of the 3x3 -> 2 convolution: one 1x1 GEMM to the 18 (tap, output) products, then a 9-tap gather
    float* taps = reinterpret_cast<float*>(x.at(ws.off_taps));
    PFB_TRY(run_conv(x, PFB_L_FLOW2T, {src_of(fh, ws.c_fh, ws.c_fh)}, PFB_EPI_LINEAR_F32, taps, 32, 0));
    PFB_TRY(pfb_flow_tap_gather(taps, 32, x.w->layers[PFB_L_FLOW2].bias, x.b->coords, flow, c->B, c->H, c->W, (pfb_stream)x.s));
  } else {
    PFB_TRY(run_conv(x, PFB_L_FLOW2, {src_of(fh, ws.c_fh, ws.c_fh)}, PFB_EPI_FLOW, flow, 2, 0));
  }
  if (fork_mask) {
    PFB_CUDA(cudaStreamWaitEvent(x.s, x.ev_join, 0));  // the upsample reads the mask
  } else if (mask_out && c->variant != 1) {
    void* mh = x.at(ws.off_mh);
    PFB_TRY(run_conv(x, PFB_L_MASK1, {src_of(x.b->net, hd, hd)}, PFB_EPI_RELU, mh, 256, 0));
    PFB_TRY(run_conv(x, PFB_L_MASK2, {src_of(mh, 256, 256)}, PFB_EPI_LINEAR, mask_out, mask_channels(c), 0, 0.25f));
  }
  return PFB_OK;
}

static int make_ctx(Ctx& x, const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                    cudaStream_t s, bool need_pyramid, bool msraft = false, bool ccmr = false) {
  PFB_TRY(check_cfg(cfg, msraft, ccmr));
  PFB_CHECK_ARG(w && buf, "raft: null weights/buffers");
  PFB_CHECK_ARG(buf->net && buf->inp && buf->coords && buf->workspace, "raft: null state buffer");
  if (need_pyramid) {
    PFB_CHECK_ARG(buf->pyramid, "raft: null pyramid");
    PFB_CHECK_ARG(!cfg->alternate_corr || (buf->fmap1 && cfg->feat_dim > 0), "raft: alternate_corr needs fmap1 and feat_dim");
  }
  x.c = cfg; x.w = w; x.b = buf; x.s = s;
  x.ws = plan(cfg);
  const size_t need = x.ws.total + (ccmr ? ccmr_plan(cfg).total : 0);
  PFB_CHECK_ARG(buf->workspace_bytes >= need, "raft: workspace %zu bytes < required %zu", buf->workspace_bytes, need);
  x.base = reinterpret_cast<char*>(buf->workspace);
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API size_t pfb_raft_workspace_bytes(const pfb_raft_cfg* cfg) {
  if (check_cfg(cfg) != PFB_OK) return 0;
  return plan(cfg).total;
}

extern "C" PFB_API int pfb_raft_update_iter(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                                    const void* corr, void* mask_out, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr));
  PFB_TRY(launch_flow_from_coords(buf->coords, reinterpret_cast<float*>(x.at(x.ws.off_flow)), cfg->B, cfg->H, cfg->W, x.s));
  PFB_TRY(run_context_terms(x));
  if (!corr) PFB_TRY(lookup(x));
  return update_iter(x, corr, mask_out);
}

// flow from the entry coordinates, the once-per-call context terms, then cfg->iters iterations (the mask head on the last one only)
static int run_iterations(Ctx& x, void* mask) {
  const pfb_raft_cfg* cfg = x.c;
  PFB_TRY(launch_flow_from_coords(x.b->coords, reinterpret_cast<float*>(x.at(x.ws.off_flow)), cfg->B, cfg->H, cfg->W, x.s));
  PFB_TRY(fork_flow_setup(x));
  if (x.side) {
    // the once-per-forward context terms ride the side stream too: they are first read by the GRU of iteration 0, after that
    // iteration's join (same stream as its flow branch, so the join covers them)
    PFB_CUDA(cudaEventRecord(x.ev_fork, x.s));
    PFB_CUDA(cudaStreamWaitEvent(x.side, x.ev_fork, 0));
    Ctx xs = x;
    xs.s = x.side;
    PFB_TRY(run_context_terms(xs));
  } else {
    PFB_TRY(run_context_terms(x));
  }
  for (int it = 0; it < cfg->iters; ++it) {
    if (x.side) {  // fork: the flow branch may start as soon as the previous iteration's coordinates are written
      PFB_CUDA(cudaEventRecord(x.ev_fork, x.s));
      PFB_CUDA(cudaStreamWaitEvent(x.side, x.ev_fork, 0));
    }
    PFB_TRY(lookup(x));
    PFB_TRY(update_iter(x, nullptr, it == cfg->iters - 1 ? mask : nullptr));
  }
  return PFB_OK;
}

extern "C" PFB_API int pfb_raft_refine(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                               pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), true));
  PFB_CHECK_ARG(buf->flow_up, "raft_refine: null flow_up");
  PFB_CHECK_ARG(cfg->variant == 1 || cfg->iters >= 1, "raft_refine: the convex upsample needs at least one iteration (mask)");
  void* mask = cfg->variant != 1 ? x.at(x.ws.off_mask) : nullptr;
  PFB_TRY(run_iterations(x, mask));
  if (cfg->variant != 1)
    return pfb_convex_upsample(buf->coords, mask, buf->flow_up, buf->flow_small, cfg->B, cfg->H, cfg->W, cfg->out_h,
                               cfg->out_w, cfg->pad_top, cfg->pad_left, cfg->dtype, stream);
  return pfb_upflow8(buf->coords, buf->flow_up, buf->flow_small, cfg->B, cfg->H, cfg->W, cfg->out_h, cfg->out_w,
                     cfg->pad_top, cfg->pad_left, stream);
}

// ---- a17: MS-RAFT+ (one call per scale of ms_raft_plus.py:177-214) ----
extern "C" PFB_API size_t pfb_msraft_workspace_bytes(const pfb_raft_cfg* cfg) {
  if (check_cfg(cfg, true) != PFB_OK) return 0;
  return plan(cfg).total;
}

extern "C" PFB_API int pfb_msraft_update_iter(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                                              const void* corr, void* mask_out, float corr_scale, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr, true));
  PFB_CHECK_ARG(corr_scale >= 0.f, "msraft_update_iter: corr_scale=%g", (double)corr_scale);
  x.corr_scale = corr_scale;
  PFB_TRY(launch_flow_from_coords(buf->coords, reinterpret_cast<float*>(x.at(x.ws.off_flow)), cfg->B, cfg->H, cfg->W, x.s));
  PFB_TRY(run_context_terms(x));
  if (!corr) PFB_TRY(lookup(x));
  return update_iter(x, corr, mask_out);
}

extern "C" PFB_API int pfb_msraft_refine(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf, float corr_scale,
                                         float* next_coords, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), true, true));
  PFB_CHECK_ARG(cfg->iters >= 1, "msraft_refine: every scale needs at least one iteration (iters=%d)", cfg->iters);
  PFB_CHECK_ARG(corr_scale >= 0.f, "msraft_refine: corr_scale=%g", (double)corr_scale);
  PFB_CHECK_ARG(next_coords || buf->flow_up, "msraft_refine: needs next_coords (coarser scales) or flow_up (the finest)");
  if (!next_coords && buf->flow_small)
    PFB_CHECK_ARG(cfg->out_h >= 16 && cfg->out_w >= 16, "msraft_refine: output %dx%d smaller than 16 px per side", cfg->out_h, cfg->out_w);
  x.corr_scale = corr_scale;
  void* mask = x.at(x.ws.off_mask);
  PFB_TRY(run_iterations(x, mask));
  if (next_coords)  // handover: the absolute coordinates, doubled and convex-upsampled with zero-padded taps (ms_raft_plus.py:198-200)
    return pfb_convex_upsample2x(buf->coords, mask, next_coords, 1, cfg->B, cfg->H, cfg->W, 0, 0, 0, 0, cfg->dtype, stream);
  PFB_TRY(pfb_convex_upsample2x(buf->coords, mask, buf->flow_up, 0, cfg->B, cfg->H, cfg->W, cfg->out_h, cfg->out_w, cfg->pad_top,
                                cfg->pad_left, cfg->dtype, stream));
  if (!buf->flow_small) return PFB_OK;
  // flow_small = downflow(flow_up, 1/16) at int(h / 16) x int(w / 16) of the un-padded size (ms_raft_plus.py:22-35, 221-224)
  const int sh = cfg->out_h / 16, sw = cfg->out_w / 16;
  return pfb_downflow(buf->flow_up, buf->flow_small, cfg->B, cfg->out_h, cfg->out_w, sh, sw, stream);
}

// ---- a18: CCMR / CCMR+ (one call per scale of ccmr.py:179-220) ----
extern "C" PFB_API size_t pfb_ccmr_workspace_bytes(const pfb_raft_cfg* cfg) {
  if (check_cfg(cfg, false, true) != PFB_OK) return 0;
  return plan(cfg).total + ccmr_plan(cfg).total;
}

static int make_ccmr_ctx(Ctx& x, const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf, cudaStream_t s,
                         bool need_pyramid, float corr_scale) {
  PFB_CHECK_ARG(w, "ccmr: null weights");
  PFB_TRY(make_ctx(x, cfg, &w->raft, buf, s, need_pyramid, false, true));
  PFB_CHECK_ARG(corr_scale >= 0.f, "ccmr: corr_scale=%g", (double)corr_scale);
  PFB_CHECK_ARG(cfg->context_dim == 128, "ccmr: the XCiT blocks expect 128 context channels");
  x.corr_scale = corr_scale;
  x.ccmr = w;
  x.ccmr_base = x.base + x.ws.total;
  return PFB_OK;
}

extern "C" PFB_API int pfb_xcit_context(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const void* inp, void* out, void* workspace,
                                        size_t workspace_bytes, pfb_stream stream) {
  PFB_CHECK_ARG(cfg && w && inp && out && workspace, "xcit_context: null pointer");
  PFB_TRY(check_cfg(cfg, false, true));
  const size_t off = plan(cfg).total, need = off + ccmr_plan(cfg).total;
  PFB_CHECK_ARG(workspace_bytes >= need, "xcit_context: workspace %zu bytes < required %zu", workspace_bytes, need);
  return ccmr_scale_setup(cfg, w, inp, out, false, reinterpret_cast<char*>(workspace) + off, as_stream(stream));
}

extern "C" PFB_API int pfb_ccmr_update_iter(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf,
                                            const void* corr, void* mask_out, float corr_scale, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ccmr_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr, corr_scale));
  PFB_TRY(ccmr_scale_setup(cfg, w, buf->inp, nullptr, true, x.ccmr_base, x.s));
  PFB_TRY(launch_flow_from_coords(buf->coords, reinterpret_cast<float*>(x.at(x.ws.off_flow)), cfg->B, cfg->H, cfg->W, x.s));
  PFB_TRY(run_context_terms(x));
  if (!corr) PFB_TRY(lookup(x));
  return update_iter(x, corr, mask_out);
}

extern "C" PFB_API int pfb_ccmr_refine(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf, float corr_scale,
                                       int upflow2, float* next_coords, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ccmr_ctx(x, cfg, w, buf, as_stream(stream), true, corr_scale));
  PFB_CHECK_ARG(cfg->iters >= 1, "ccmr_refine: every scale needs at least one iteration (iters=%d)", cfg->iters);
  PFB_CHECK_ARG(upflow2 == 0 || upflow2 == 1, "ccmr_refine: upflow2=%d (0 or 1)", upflow2);
  PFB_CHECK_ARG(next_coords || buf->flow_up, "ccmr_refine: needs next_coords (coarser scales) or flow_up (the finest)");
  if (!next_coords) {
    const int f = 2 << upflow2;  // the output grid is f times this scale's
    PFB_CHECK_ARG(cfg->out_h > 0 && cfg->out_w > 0 && cfg->pad_top >= 0 && cfg->pad_left >= 0 && cfg->out_h + cfg->pad_top <= f * cfg->H &&
                      cfg->out_w + cfg->pad_left <= f * cfg->W,
                  "ccmr_refine: output window %dx%d+(%d,%d) outside %dx%d", cfg->out_h, cfg->out_w, cfg->pad_top, cfg->pad_left, f * cfg->H,
                  f * cfg->W);
    if (buf->flow_small)
      PFB_CHECK_ARG(cfg->out_h >= 16 && cfg->out_w >= 16, "ccmr_refine: output %dx%d smaller than 16 px per side", cfg->out_h, cfg->out_w);
  }
  PFB_TRY(ccmr_scale_setup(cfg, w, buf->inp, nullptr, true, x.ccmr_base, x.s));
  void* mask = x.at(x.ws.off_mask);
  PFB_TRY(run_iterations(x, mask));
  if (next_coords)  // handover: the convex 2x of the FLOW on the next scale's grid (ccmr.py:195-202)
    return pfb_convex_handover2x(buf->coords, mask, next_coords, cfg->B, cfg->H, cfg->W, cfg->dtype, stream);
  return ccmr_output(cfg, buf->coords, mask, buf->flow_up, buf->flow_small, upflow2, x.ccmr_base, x.s);
}
