// SEA-RAFT's refinement loop (ptlflow/models/sea_raft/sea_raft.py:189-236, update.py:18-54, layer.py:41-83): init_conv and the
// initial flow head, then `iters` times lookup -> RAFT's motion encoder -> num_blocks ConvNeXt blocks -> flow head, then the mask
// head and the convex upsample once.  Every stage is a launch of this library's kernels on the caller's stream, so the whole loop
// is one CUDA graph when the host captures it.  The lookup, the motion encoder, the flow head, the mask head and flow-from-coords
// are the raft loop's (refine.cuh).
//
// Layout: one [P][384] buffer X = [net | context | motion (126) | flow (2)] that every producer writes at its column offset:
// init_conv writes net | context, the motion encoder's last layer motion and the flow, each ConvNeXt block the new net.  X is at
// once the depthwise input of a block and the second source of its output layer, so no concatenation is ever copied.
#include "refine.cuh"

namespace pfb {
namespace {

constexpr int kX = 384;    // [net | context | motion | flow]
constexpr int kHid = 512;  // ConvNeXt hidden width, 4 * 128

struct SrWs {
  int planes, corr_stride;
  size_t off_corr, off_cor1, off_corflo, off_flo1, off_x, off_xn, off_h, off_net, off_fh, off_taps, off_mh, off_mask, off_flow,
      off_flags, total;
};

SrWs plan(const pfb_raft_cfg* c) {
  SrWs w{};
  const size_t P = (size_t)c->B * c->H * c->W, es = dtype_size(c->dtype);
  const int K = 2 * c->corr_radius + 1;
  w.planes = c->corr_levels * K * K;
  w.corr_stride = c->dtype == PFB_F32 ? w.planes : (int)align_up(w.planes, 8);
  const size_t loop = c->iters > 0 ? 1 : 0;  // iters = 0: no lookup, no motion encoder, no ConvNeXt block
  Carve k;
  w.off_corr = k.take(loop * P * w.corr_stride * es);
  w.off_cor1 = k.take(loop * P * 256 * es);
  w.off_corflo = k.take(loop * P * 256 * es);
  w.off_flo1 = k.take(loop * P * 128 * es);
  w.off_x = k.take(P * kX * es);
  w.off_xn = k.take(loop * P * kX * es);
  w.off_h = k.take(loop * P * kHid * es);
  w.off_net = k.take(loop * P * 128 * es);
  w.off_fh = k.take(P * 256 * es);
  w.off_taps = k.take(P * 32 * sizeof(float));
  w.off_mh = k.take(P * 256 * es);
  w.off_mask = k.take(P * 576 * es);
  w.off_flow = k.take(P * 2 * sizeof(float));
  w.off_flags = k.take(c->alternate_corr ? P : 0);
  w.total = k.total;
  return w;
}

int check_cfg(const pfb_raft_cfg* c) {
  PFB_TRY(check_loop_cfg(c, "searaft", c && c->iters > 0));  // iters = 0 looks nothing up
  PFB_CHECK_ARG(c->variant == PFB_VARIANT_SEA_RAFT, "searaft: variant=%d (the sea_raft loop is PFB_VARIANT_SEA_RAFT)", c->variant);
  PFB_CHECK_ARG(c->hidden_dim == 128 && c->context_dim == 128, "searaft: the update block expects hidden=context=128");
  return PFB_OK;
}

int check_layer(const pfb_layer& L, int cin, int cout, const char* name) {
  PFB_CHECK_ARG(L.weight && L.Cin == cin && L.Cout == cout, "searaft: layer %s must be %d -> %d (has %d -> %d)", name, cin, cout,
                L.Cin, L.Cout);
  return PFB_OK;
}

int check_weights(const pfb_raft_cfg* c, const pfb_searaft_weights* w, const SrWs& ws) {
  PFB_CHECK_ARG(w, "searaft: null weights");
  PFB_TRY(check_layer(w->init_conv, 256, 256, "init_conv"));
  PFB_TRY(check_layer(w->flow1, 128, 256, "flow_head.0"));
  PFB_TRY(check_layer(w->flow2, 256, 2, "flow_head.2"));
  PFB_TRY(check_layer(w->mask1, 128, 256, "upsample_weight.0"));
  PFB_TRY(check_layer(w->mask2, 256, 576, "upsample_weight.2"));
  if (c->iters == 0) return PFB_OK;
  PFB_TRY(check_layer(w->convc1, ws.planes, 256, "convc1"));
  PFB_TRY(check_layer(w->convc2, 256, 192, "convc2"));
  PFB_TRY(check_layer(w->convf1, 2, 128, "convf1"));
  PFB_TRY(check_layer(w->convf2, 128, 64, "convf2"));
  PFB_TRY(check_layer(w->conv, 256, 126, "conv"));
  PFB_CHECK_ARG(w->num_blocks >= 1 && w->num_blocks <= PFB_SR_MAX_BLOCKS && w->ln_eps > 0.f, "searaft: num_blocks=%d ln_eps=%g",
                w->num_blocks, (double)w->ln_eps);
  for (int i = 0; i < w->num_blocks; ++i) {
    const pfb_convnext_block& k = w->blocks[i];
    PFB_CHECK_ARG(k.dw_weight && k.dw_bias && (k.dw_k & 1) && k.dw_k >= 1, "searaft: block %d depthwise filter (k=%d)", i, k.dw_k);
    PFB_TRY(check_layer(k.pw1, kX, kHid, "pwconv1"));
    PFB_TRY(check_layer(k.out, kHid + kX, 128, "final"));
  }
  return PFB_OK;
}

struct SrCtx {
  const pfb_raft_cfg* c;
  const pfb_searaft_weights* w;
  const pfb_raft_buffers* b;
  SrWs ws;
  char* base;
  cudaStream_t s;
  ConvExtras e;  // every layer's coordinates and flow
  void* at(size_t off) const { return base + off; }
  float* flow() const { return reinterpret_cast<float*>(base + ws.off_flow); }
};

// flow_head(net)[:, :2] (sea_raft.py:195, 225): coords += delta, flow = coords - grid
int flow_head(const SrCtx& x) {
  return pfb::flow_head(x.c, x.s, x.e, x.w->flow1, x.w->flow2, &x.w->flow2t, src_of(x.at(x.ws.off_x), 128, kX), x.at(x.ws.off_fh), 256,
                        reinterpret_cast<float*>(x.at(x.ws.off_taps)), x.flow());
}

// 0.25 * upsample_weight(net) (sea_raft.py:226)
int mask_head(const SrCtx& x, void* mask_out) {
  return pfb::mask_head(x.c, x.s, x.e, x.w->mask1, x.w->mask2, src_of(x.at(x.ws.off_x), 128, kX), x.at(x.ws.off_mh), mask_out, 576);
}

// BasicUpdateBlock (update.py:49-54) on X, whose net | context columns are current, + the flow head
int update_iter(const SrCtx& x, const void* corr_ext, void* mask_out) {
  const pfb_raft_cfg* c = x.c;
  const SrWs& ws = x.ws;
  const pfb_searaft_weights* w = x.w;
  const size_t es = dtype_size(c->dtype), P = (size_t)c->B * c->H * c->W;
  const void* corr = corr_ext ? corr_ext : x.at(ws.off_corr);
  const int corr_stride = corr_ext ? ws.planes : ws.corr_stride;
  char* X = reinterpret_cast<char*>(x.at(ws.off_x));
  // ---- motion encoder (update.py:28-36): writes X[:, 256:384] = [relu(conv(cor | flo)) | flow] ----
  const MotionLayers ml{&w->convc1, &w->convc2, &w->convf1, &w->convf2, &w->conv};
  const MotionBuffers mb{x.at(ws.off_cor1), x.at(ws.off_corflo), x.at(ws.off_flo1), 256, 192, 128, 64};
  PFB_TRY(motion_encoder(c, x.s, x.e, ml, mb, src_of(corr, ws.planes, corr_stride), {PFB_EPI_RELU_APPEND_FLOW, X, kX, 256}));
  // ---- num_blocks ConvNextBlocks, net = final(x + gamma * pwconv2(gelu(pwconv1(LN(dwconv(x)))))) (layer.py:71-83) ----
  void* xn = x.at(ws.off_xn);
  void* h = x.at(ws.off_h);
  void* net = x.at(ws.off_net);
  for (int i = 0; i < w->num_blocks; ++i) {
    const pfb_convnext_block& k = w->blocks[i];
    PFB_TRY(pfb_depthwise_conv_layernorm(X, kX, 0, xn, kX, 0, k.dw_weight, k.dw_bias, c->B, c->H, c->W, kX, k.dw_k, w->ln_eps, c->dtype,
                                         (pfb_stream)x.s));
    PFB_TRY(launch_conv(c, x.s, k.pw1, {src_of(xn, kX, kX)}, {PFB_EPI_GELU, h, kHid, 0}, x.e));
    // pwconv2, gamma, the residual and final as one GEMM over [h | x].  The new net goes to its own buffer and is copied into X
    // afterwards: the layer reads all of X, and on the SIMT kernel the CTAs of output columns 64..127 may still be reading the
    // net columns of a pixel when those of columns 0..63 write them.
    PFB_TRY(launch_conv(c, x.s, k.out, {src_of(h, kHid, kHid), src_of(X, kX, kX)}, {PFB_EPI_LINEAR, net, 128, 0}, x.e));
    PFB_CUDA(cudaMemcpy2DAsync(X, kX * es, net, 128 * es, 128 * es, P, cudaMemcpyDeviceToDevice, x.s));
  }
  // ---- flow head, coords += delta (sea_raft.py:225-227) ----
  PFB_TRY(flow_head(x));
  if (mask_out) PFB_TRY(mask_head(x, mask_out));
  return PFB_OK;
}

int make_ctx(SrCtx& x, const pfb_raft_cfg* cfg, const pfb_searaft_weights* w, const pfb_raft_buffers* buf, cudaStream_t s,
             bool need_pyramid) {
  PFB_TRY(check_cfg(cfg));
  x.c = cfg; x.w = w; x.b = buf; x.s = s;
  x.ws = plan(cfg);
  PFB_TRY(check_loop_buffers(cfg, buf, need_pyramid, x.ws.total, "searaft"));
  PFB_TRY(check_weights(cfg, w, x.ws));
  x.base = reinterpret_cast<char*>(buf->workspace);
  x.e.coords = buf->coords; x.e.flow = x.flow();
  return PFB_OK;
}

int lookup(const SrCtx& x) {
  return raft_lookup(x.c, x.b->pyramid, x.b->fmap1, x.b->coords, x.at(x.ws.off_corr), x.ws.corr_stride, x.at(x.ws.off_flags), x.s);
}

}  // namespace
}  // namespace pfb

using namespace pfb;

extern "C" PFB_API size_t pfb_searaft_workspace_bytes(const pfb_raft_cfg* cfg) {
  if (check_cfg(cfg) != PFB_OK) return 0;
  return plan(cfg).total;
}

extern "C" PFB_API int pfb_searaft_update_iter(const pfb_raft_cfg* cfg, const pfb_searaft_weights* w, const pfb_raft_buffers* buf,
                                               const void* corr, void* mask_out, pfb_stream stream) {
  SrCtx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr));
  PFB_CHECK_ARG(cfg->iters >= 1, "searaft_update_iter: cfg->iters must be >= 1 (the update block's weights are read)");
  PFB_TRY(copy_wide_state(cfg, buf, x.at(x.ws.off_x), kX, true, x.s));
  PFB_TRY(launch_flow_from_coords(buf->coords, x.flow(), cfg->B, cfg->H, cfg->W, x.s));
  if (!corr) PFB_TRY(lookup(x));
  PFB_TRY(update_iter(x, corr, mask_out));
  return copy_wide_state(cfg, buf, x.at(x.ws.off_x), kX, false, x.s);  // the final net
}

extern "C" PFB_API int pfb_searaft_refine(const pfb_raft_cfg* cfg, const pfb_searaft_weights* w, const pfb_raft_buffers* buf,
                                          pfb_stream stream) {
  SrCtx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), cfg && cfg->iters > 0));
  PFB_CHECK_ARG(buf->flow_up, "searaft_refine: null flow_up");
  // net | context = init_conv(cnet) straight into X (sea_raft.py:190-192), then the initial flow (sea_raft.py:195-198)
  PFB_TRY(launch_conv(cfg, x.s, w->init_conv, {src_of(buf->inp, 256, 256)}, {PFB_EPI_LINEAR, x.at(x.ws.off_x), kX, 0}, x.e));
  PFB_TRY(flow_head(x));
  void* mask = x.at(x.ws.off_mask);
  for (int it = 0; it < cfg->iters; ++it) {
    PFB_TRY(lookup(x));
    PFB_TRY(update_iter(x, nullptr, nullptr));
  }
  PFB_TRY(mask_head(x, mask));  // only the last prediction is returned in eval (sea_raft.py:274)
  PFB_TRY(copy_wide_state(cfg, buf, x.at(x.ws.off_x), kX, false, x.s));
  return pfb_convex_upsample(buf->coords, mask, buf->flow_up, buf->flow_small, cfg->B, cfg->H, cfg->W, cfg->out_h, cfg->out_w,
                             cfg->pad_top, cfg->pad_left, cfg->dtype, stream);
}
