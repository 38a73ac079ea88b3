// SKFlow's refinement loop (ptlflow/models/skflow/skflow.py:197-232, update.py:7-99): lookup -> large-kernel motion encoder ->
// GMA aggregate -> PCBlock "GRU" -> PCBlock flow head, `iters` times, then the mask head and the convex upsample once.
// Every stage is a launch of this library's kernels on the caller's stream, so the whole loop is one CUDA graph when the host
// captures it.  The lookup, the attention aggregate, flow-from-coords and the upsample are the raft / gma loop's (refine.cuh).
//
// Layout: one [P][512] buffer X = [net | inp | motion | motion_global] that every producer writes at its column offset: the
// motion encoder's last layer writes motion (126 channels + the flow), the aggregate motion_global, the update block the new net.
// X is at the same time the update block's input and its ffn1 residual, so no concatenation is ever copied.  Inside a PCBlock
// the activations ping-pong between two scratch buffers; channel counts are padded to multiples of 32 whose padding stays zero.
#include "refine.cuh"

#define PFB_TRY(expr)        \
  do {                       \
    int rc__ = (expr);       \
    if (rc__ != PFB_OK) return rc__; \
  } while (0)

namespace pfb {
namespace {

constexpr int kX = 512;  // [net | inp | motion | motion_global]

int heads_sk(const pfb_raft_cfg* c) { return c->num_heads > 0 ? c->num_heads : 1; }
int planes_of(const pfb_raft_cfg* c) { const int K = 2 * c->corr_radius + 1; return c->corr_levels * K * K; }

struct SkWs {
  int planes, corr_stride, cmax, hmax, n_pad;
  size_t off_corr, off_cor1, off_corflo, off_flo1, off_x, off_a, off_b, off_h, off_mh, off_mask, off_flow, off_vbuf, off_vT, off_agg,
      off_flags, total;
};

SkWs plan(const pfb_raft_cfg* c) {
  SkWs w{};
  const size_t P = (size_t)c->B * c->H * c->W, es = dtype_size(c->dtype), vdim = (size_t)heads_sk(c) * 128;
  w.planes = planes_of(c);
  w.corr_stride = (int)align_up(w.planes, 32);
  w.cmax = w.corr_stride > kX ? w.corr_stride : kX;
  const int hid_c1 = (int)align_up((size_t)(3 * w.planes) / 2, 32);
  w.hmax = hid_c1 > 3 * kX / 2 ? hid_c1 : 3 * kX / 2;
  w.n_pad = (int)align_up((size_t)c->H * c->W, 64);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  w.off_corr = take(P * w.corr_stride * es);
  w.off_cor1 = take(P * 256 * es);
  w.off_corflo = take(P * 256 * es);
  w.off_flo1 = take(P * 128 * es);
  w.off_x = take(P * kX * es);
  w.off_a = take(P * w.cmax * es);
  w.off_b = take(P * w.cmax * es);
  w.off_h = take(P * w.hmax * es);
  w.off_mh = take(P * 256 * es);
  w.off_mask = take(P * 576 * es);
  w.off_flow = take(P * 2 * sizeof(float));
  w.off_vbuf = take(P * vdim * es);
  w.off_vT = take((size_t)c->B * vdim * w.n_pad * es);
  w.off_agg = take(vdim > 128 ? P * vdim * es : 0);
  w.off_flags = take(c->alternate_corr ? P : 0);
  w.total = off;
  return w;
}

int check_cfg(const pfb_raft_cfg* c) {
  PFB_CHECK_ARG(c, "skflow: null cfg");
  PFB_CHECK_ARG(c->variant == 3, "skflow: variant=%d (the skflow loop is variant 3)", c->variant);
  PFB_CHECK_ARG(dtype_ok(c->dtype), "skflow: bad dtype");
  PFB_CHECK_ARG(c->B > 0 && c->H > 0 && c->W > 0, "skflow: bad grid %dx%dx%d", c->B, c->H, c->W);
  PFB_CHECK_ARG(c->corr_levels >= 1 && c->corr_levels <= PFB_MAX_LEVELS && c->corr_radius >= 0 && c->corr_radius <= 15,
                "skflow: corr_levels=%d corr_radius=%d", c->corr_levels, c->corr_radius);
  PFB_CHECK_ARG((c->H >> (c->corr_levels - 1)) >= 1 && (c->W >> (c->corr_levels - 1)) >= 1,
                "skflow: %dx%d grid too small for %d levels", c->H, c->W, c->corr_levels);
  PFB_CHECK_ARG(c->hidden_dim == 128 && c->context_dim == 128 && c->iters >= 0, "skflow: the update block expects hidden=context=128");
  PFB_CHECK_ARG(c->num_heads >= 0 && c->num_heads <= 64, "skflow: num_heads=%d", c->num_heads);
  PFB_CHECK_ARG(c->volume_layout == 0 || (c->volume_layout == 1 && c->dtype != PFB_F32 && !c->alternate_corr && c->corr_levels <= 4),
                "skflow: volume_layout=%d needs f16/bf16, a materialised pyramid and <= 4 levels", c->volume_layout);
  return PFB_OK;
}

int check_block(const pfb_pc_block& k, int C, int cout, int hmax, const char* name) {
  PFB_CHECK_ARG(k.C == C && k.hid > 0 && k.hid <= hmax && k.hid % 2 == 0, "skflow: block %s has C=%d hid=%d (expected C=%d, hid <= %d)",
                name, k.C, k.hid, C, hmax);
  PFB_CHECK_ARG(k.ffn1a.weight && k.ffn1b.weight && k.pw.weight && k.ffn2a.weight && k.ffn2b.weight, "skflow: block %s lacks a layer", name);
  PFB_CHECK_ARG(k.ffn1a.Cin == C && k.ffn1a.Cout == k.hid && k.ffn1b.Cin == k.hid && k.ffn1b.Cout == C && k.pw.Cin == C && k.pw.Cout == C &&
                    k.ffn2a.Cin == C && k.ffn2a.Cout == k.hid && k.ffn2b.Cin == k.hid && k.ffn2b.Cout == cout,
                "skflow: block %s layer shapes do not chain (C=%d hid=%d out=%d)", name, C, k.hid, cout);
  PFB_CHECK_ARG(k.n_dw >= 0 && k.n_dw <= PFB_SK_MAX_DW, "skflow: block %s has %d depthwise steps", name, k.n_dw);
  for (int i = 0; i < k.n_dw; ++i)
    PFB_CHECK_ARG((k.dw_k[i] & 1) && k.dw_k[i] >= 1 && k.dw_k[i] <= 31 && k.dw_weight[i] && k.dw_bias[i],
                  "skflow: block %s depthwise step %d (k=%d)", name, i, k.dw_k[i]);
  return PFB_OK;
}

int check_weights(const pfb_raft_cfg* c, const pfb_skflow_weights* w, const SkWs& ws) {
  PFB_CHECK_ARG(w, "skflow: null weights");
  const pfb_pc_block* b = w->blocks;
  PFB_TRY(check_block(b[PFB_SK_CONVC1], ws.corr_stride, 256, ws.hmax, "convc1"));
  PFB_TRY(check_block(b[PFB_SK_CONVC2], 256, 192, ws.hmax, "convc2"));
  PFB_TRY(check_block(b[PFB_SK_CONVF2], 128, 64, ws.hmax, "convf2"));
  PFB_TRY(check_block(b[PFB_SK_CONV], 256, 126, ws.hmax, "conv"));
  PFB_TRY(check_block(b[PFB_SK_GRU], kX, 128, ws.hmax, "gru"));
  PFB_TRY(check_block(b[PFB_SK_FLOW_HEAD], 128, 2, ws.hmax, "flow_head"));
  PFB_CHECK_ARG(w->convf1.weight && w->convf1.Cin == 2 && w->convf1.Cout == 128 && w->convf1.KH == 1 && w->convf1.KW == 1,
                "skflow: convf1 must be a 1x1 2 -> 128 layer");
  PFB_CHECK_ARG(w->mask1.weight && w->mask2.weight && w->mask1.Cin == 128 && w->mask2.Cout == 576, "skflow: mask head missing");
  (void)c;
  return PFB_OK;
}

struct SkCtx {
  const pfb_raft_cfg* c;
  const pfb_skflow_weights* w;
  const pfb_raft_buffers* b;
  SkWs ws;
  char* base;
  cudaStream_t s;
  void* at(size_t off) const { return base + off; }
  float* flow() const { return reinterpret_cast<float*>(base + ws.off_flow); }
};

pfb_conv_src src_of(const void* ptr, int channels, int stride, int offset = 0, int is_f32 = 0) {
  pfb_conv_src s;
  s.ptr = ptr; s.channels = channels; s.stride = stride; s.offset = offset; s.is_f32 = is_f32;
  return s;
}

struct Out {
  int epi;
  void* ptr;
  int stride, offset;
  float scale;
};

int conv(const SkCtx& x, const pfb_layer& L, const pfb_conv_src& src, const Out& o, const pfb_conv_src* res = nullptr,
         const float* post_w = nullptr, const float* post_b = nullptr) {
  PFB_CHECK_ARG(L.weight && src.channels == L.Cin, "skflow: layer expects Cin=%d, source provides %d", L.Cin, src.channels);
  pfb_conv_params p{};
  p.src[0] = src;
  p.nsrc = 1;
  p.B = x.c->B; p.H = x.c->H; p.W = x.c->W;
  p.KH = L.KH; p.KW = L.KW; p.Cout = L.Cout; p.Cout_pad = L.Cout_pad;
  p.weight = L.weight; p.bias = L.bias;
  p.epilogue = o.epi; p.scale = o.scale;
  p.out = o.ptr; p.out_stride = o.stride; p.out_offset = o.offset;
  p.coords = x.b->coords; p.flow = x.flow();
  p.dtype = x.c->dtype; p.impl = x.c->impl;
  p.weight_k = L.weight_k; p.Cin_pad = L.Cin_pad; p.Cout_pad_k = L.Cout_pad_k;
  if (res) {
    p.residual = res->ptr; p.residual_stride = res->stride; p.residual_offset = res->offset;
    p.post_w = post_w; p.post_b = post_b;
  }
  return pfb_conv2d(&p, (pfb_stream)x.s);
}

// PCBlock4_Deep_nopool_res (update.py:7-41) on `in` (k.C channels); the last layer's output and epilogue are the caller's
int pc_block(const SkCtx& x, const pfb_pc_block& k, const pfb_conv_src& in, const Out& last) {
  char* h = reinterpret_cast<char*>(x.at(x.ws.off_h));
  char* cur = reinterpret_cast<char*>(x.at(x.ws.off_a));
  char* oth = reinterpret_cast<char*>(x.at(x.ws.off_b));
  const int C = k.C, hid = k.hid;
  // x = gelu(x + ffn1(x)); a leading k = 1 entry of k_conv, gelu(x + w * x + b), rides the same epilogue
  PFB_TRY(conv(x, k.ffn1a, in, Out{PFB_EPI_GELU, h, hid, 0, 1.f}));
  int first = 0;
  const float *pw = nullptr, *pb = nullptr;
  if (k.n_dw > 0 && k.dw_k[0] == 1) { pw = k.dw_weight[0]; pb = k.dw_bias[0]; first = 1; }
  PFB_TRY(conv(x, k.ffn1b, src_of(h, hid, hid), Out{PFB_EPI_RESIDUAL_GELU, cur, C, 0, 1.f}, &in, pw, pb));
  // x = gelu(x + dw_k(x)) for the remaining entries of k_conv
  for (int i = first; i < k.n_dw; ++i) {
    PFB_TRY(pfb_depthwise_conv_gelu(cur, C, 0, oth, C, 0, k.dw_weight[i], k.dw_bias[i], x.c->B, x.c->H, x.c->W, C, k.dw_k[i], x.c->dtype,
                                    (pfb_stream)x.s));
    char* t = cur; cur = oth; oth = t;
  }
  // x = gelu(x + pw(x))
  const pfb_conv_src xs = src_of(cur, C, C);
  PFB_TRY(conv(x, k.pw, xs, Out{PFB_EPI_RESIDUAL_GELU, oth, C, 0, 1.f}, &xs));
  // out = ffn2(x)
  PFB_TRY(conv(x, k.ffn2a, src_of(oth, C, C), Out{PFB_EPI_GELU, h, hid, 0, 1.f}));
  return conv(x, k.ffn2b, src_of(h, hid, hid), last);
}

// One SKUpdateBlock6_Deep_nopoolres_AllDecoder evaluation + the coordinate update (update.py:81-99, skflow.py:211-218)
int update_iter(const SkCtx& x, const void* corr_ext, void* mask_out) {
  const pfb_raft_cfg* c = x.c;
  const SkWs& ws = x.ws;
  const pfb_pc_block* blk = x.w->blocks;
  const void* corr = corr_ext ? corr_ext : x.at(ws.off_corr);
  void* cor1 = x.at(ws.off_cor1);
  void* corflo = x.at(ws.off_corflo);
  void* flo1 = x.at(ws.off_flo1);
  void* X = x.at(ws.off_x);
  // ---- motion encoder (update.py:53-61) ----
  PFB_TRY(pc_block(x, blk[PFB_SK_CONVC1], src_of(corr, ws.corr_stride, ws.corr_stride), Out{PFB_EPI_GELU, cor1, 256, 0, 1.f}));
  PFB_TRY(pc_block(x, blk[PFB_SK_CONVC2], src_of(cor1, 256, 256), Out{PFB_EPI_LINEAR, corflo, 256, 0, 1.f}));
  PFB_TRY(conv(x, x.w->convf1, src_of(x.flow(), 2, 2, 0, 1), Out{PFB_EPI_LINEAR, flo1, 128, 0, 1.f}));
  PFB_TRY(pc_block(x, blk[PFB_SK_CONVF2], src_of(flo1, 128, 128), Out{PFB_EPI_LINEAR, corflo, 256, 192, 1.f}));
  PFB_TRY(pc_block(x, blk[PFB_SK_CONV], src_of(corflo, 256, 256), Out{PFB_EPI_LINEAR_APPEND_FLOW, X, kX, 256, 1.f}));
  // ---- motion_global = Aggregate(attention, motion) (update.py:90) ----
  PFB_TRY(gma_aggregate(c, x.w->agg_v, x.w->agg_proj, x.b->attention, x.b->agg_gamma, X, kX, 256, 384, x.at(ws.off_vbuf), x.at(ws.off_vT),
                        x.at(ws.off_agg), ws.n_pad, x.s));
  // ---- net = gru(cat[net, inp, motion, motion_global]): linear, no gates (update.py:94) ----
  PFB_TRY(pc_block(x, blk[PFB_SK_GRU], src_of(X, kX, kX), Out{PFB_EPI_LINEAR, X, kX, 0, 1.f}));
  // ---- delta = flow_head(net); coords += delta (update.py:96, skflow.py:218) ----
  PFB_TRY(pc_block(x, blk[PFB_SK_FLOW_HEAD], src_of(X, 128, kX), Out{PFB_EPI_FLOW, x.flow(), 2, 0, 1.f}));
  if (mask_out) {  // mask = 0.25 * mask(net) (update.py:98-99)
    void* mh = x.at(ws.off_mh);
    PFB_TRY(conv(x, x.w->mask1, src_of(X, 128, kX), Out{PFB_EPI_RELU, mh, 256, 0, 1.f}));
    PFB_TRY(conv(x, x.w->mask2, src_of(mh, 256, 256), Out{PFB_EPI_LINEAR, mask_out, 576, 0, 0.25f}));
  }
  return PFB_OK;
}

int make_ctx(SkCtx& x, const pfb_raft_cfg* cfg, const pfb_skflow_weights* w, const pfb_raft_buffers* buf, cudaStream_t s,
             bool need_pyramid) {
  PFB_TRY(check_cfg(cfg));
  PFB_CHECK_ARG(buf, "skflow: null buffers");
  PFB_CHECK_ARG(buf->net && buf->inp && buf->coords && buf->workspace && buf->attention, "skflow: null state buffer / attention");
  if (need_pyramid) {
    PFB_CHECK_ARG(buf->pyramid, "skflow: null pyramid");
    PFB_CHECK_ARG(!cfg->alternate_corr || (buf->fmap1 && cfg->feat_dim > 0), "skflow: alternate_corr needs fmap1 and feat_dim");
  }
  x.c = cfg; x.w = w; x.b = buf; x.s = s;
  x.ws = plan(cfg);
  PFB_TRY(check_weights(cfg, w, x.ws));
  PFB_CHECK_ARG(buf->workspace_bytes >= x.ws.total, "skflow: workspace %zu bytes < required %zu", buf->workspace_bytes, x.ws.total);
  x.base = reinterpret_cast<char*>(buf->workspace);
  return PFB_OK;
}

// net -> X[:, 0:128], inp -> X[:, 128:256]; the flow of the current coordinates; zero lookup columns past the planes
int begin(const SkCtx& x, bool lookup_buffer) {
  const pfb_raft_cfg* c = x.c;
  const size_t es = dtype_size(c->dtype), P = (size_t)c->B * c->H * c->W;
  char* X = reinterpret_cast<char*>(x.at(x.ws.off_x));
  PFB_CUDA(cudaMemcpy2DAsync(X, kX * es, x.b->net, 128 * es, 128 * es, P, cudaMemcpyDeviceToDevice, x.s));
  PFB_CUDA(cudaMemcpy2DAsync(X + 128 * es, kX * es, x.b->inp, 128 * es, 128 * es, P, cudaMemcpyDeviceToDevice, x.s));
  if (lookup_buffer) PFB_CUDA(cudaMemsetAsync(x.at(x.ws.off_corr), 0, P * x.ws.corr_stride * es, x.s));
  return launch_flow_from_coords(x.b->coords, x.flow(), c->B, c->H, c->W, x.s);
}

int finish(const SkCtx& x) {  // the final hidden state back to buf->net
  const size_t es = dtype_size(x.c->dtype), P = (size_t)x.c->B * x.c->H * x.c->W;
  PFB_CUDA(cudaMemcpy2DAsync(x.b->net, 128 * es, x.at(x.ws.off_x), kX * es, 128 * es, P, cudaMemcpyDeviceToDevice, x.s));
  return PFB_OK;
}

int lookup(const SkCtx& x) {
  return raft_lookup(x.c, x.b->pyramid, x.b->fmap1, x.b->coords, x.at(x.ws.off_corr), x.ws.corr_stride, x.at(x.ws.off_flags), x.s);
}

}  // namespace
}  // namespace pfb

using namespace pfb;

extern "C" PFB_API size_t pfb_skflow_workspace_bytes(const pfb_raft_cfg* cfg) {
  if (check_cfg(cfg) != PFB_OK) return 0;
  return plan(cfg).total;
}

extern "C" PFB_API int pfb_skflow_update_iter(const pfb_raft_cfg* cfg, const pfb_skflow_weights* w, const pfb_raft_buffers* buf,
                                              const void* corr, void* mask_out, pfb_stream stream) {
  SkCtx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr));
  PFB_TRY(begin(x, corr == nullptr));
  if (!corr) PFB_TRY(lookup(x));
  PFB_TRY(update_iter(x, corr, mask_out));
  return finish(x);
}

extern "C" PFB_API int pfb_skflow_refine(const pfb_raft_cfg* cfg, const pfb_skflow_weights* w, const pfb_raft_buffers* buf,
                                         pfb_stream stream) {
  SkCtx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), true));
  PFB_CHECK_ARG(buf->flow_up, "skflow_refine: null flow_up");
  PFB_CHECK_ARG(cfg->iters >= 1, "skflow_refine: the convex upsample needs at least one iteration (mask)");
  PFB_TRY(begin(x, true));
  void* mask = x.at(x.ws.off_mask);
  for (int it = 0; it < cfg->iters; ++it) {
    PFB_TRY(lookup(x));
    PFB_TRY(update_iter(x, nullptr, it == cfg->iters - 1 ? mask : nullptr));
  }
  PFB_TRY(finish(x));
  return pfb_convex_upsample(buf->coords, mask, buf->flow_up, buf->flow_small, cfg->B, cfg->H, cfg->W, cfg->out_h, cfg->out_w,
                             cfg->pad_top, cfg->pad_left, cfg->dtype, stream);
}
