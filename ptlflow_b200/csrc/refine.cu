// Host-side orchestration of the refinement loop: lookup -> motion encoder -> GRU -> heads,
// `iters` times, then the upsample.  Mirrors the data flow of
//   ptlflow/models/raft/raft.py:170-192 and ptlflow/models/raft/update.py:115-153
// but every stage is one launch of this library's kernels on the caller's stream (so the whole
// loop can be captured in a CUDA graph by the host), no torch.cat / permute copies exist, and
// the mask head + upsample run once (eval returns only the last prediction, raft.py:192).
#include <stdlib.h>

#include "refine.cuh"

namespace pfb {

// ---- shared by every loop (refine.cuh) ----

int launch_conv(const pfb_raft_cfg* c, cudaStream_t s, const pfb_layer& L, std::initializer_list<pfb_conv_src> srcs, const ConvOut& o,
                const ConvExtras& e) {
  pfb_conv_params p{};
  int cin = 0;
  for (const auto& src : srcs) { p.src[p.nsrc++] = src; cin += src.channels; }
  PFB_CHECK_ARG(L.weight, "conv: a %dx%d %d -> %d layer has no packed weight", L.KH, L.KW, L.Cin, L.Cout);
  // the lookup buffer may be wider than the layer's real Cin (zero pad columns <-> zero weight rows)
  PFB_CHECK_ARG(cin == L.Cin, "conv: a %dx%d %d -> %d layer expects Cin=%d, sources provide %d", L.KH, L.KW, L.Cin, L.Cout, L.Cin, cin);
  p.B = e.B > 0 ? e.B : c->B; p.H = c->H; p.W = c->W;
  p.KH = L.KH; p.KW = L.KW; p.Cout = L.Cout; p.Cout_pad = L.Cout_pad;
  p.weight = L.weight; p.bias = L.bias;
  p.weight_k = L.weight_k; p.Cin_pad = L.Cin_pad; p.Cout_pad_k = L.Cout_pad_k;
  p.epilogue = o.epi; p.scale = o.scale;
  p.out = o.ptr; p.out_stride = o.stride; p.out_offset = o.offset;
  p.aux_h = e.aux_h; p.aux_z = e.aux_z; p.hidden = e.hidden;
  p.coords = e.coords; p.flow = e.flow;
  p.addend = e.addend; p.addend_stride = e.addend_stride;
  if (e.residual) { p.residual = e.residual->ptr; p.residual_stride = e.residual->stride; p.residual_offset = e.residual->offset; }
  p.post_w = e.post_w; p.post_b = e.post_b;
  p.w_rows_per_sample = e.w_rows_per_sample;
  p.dtype = c->dtype; p.impl = e.impl >= 0 ? e.impl : c->impl;
  return pfb_conv2d(&p, (pfb_stream)s);
}

int check_loop_cfg(const pfb_raft_cfg* c, const char* name, bool levels_fit_grid, int max_radius, int pool_min_side) {
  PFB_CHECK_ARG(c, "%s: null cfg", name);
  PFB_CHECK_ARG(dtype_ok(c->dtype), "%s: bad dtype %d", name, (int)c->dtype);
  PFB_CHECK_ARG(c->B > 0 && c->H > 0 && c->W > 0, "%s: bad grid %dx%dx%d", name, c->B, c->H, c->W);
  PFB_CHECK_ARG(c->corr_levels >= 1 && c->corr_levels <= PFB_MAX_LEVELS && c->corr_radius >= 0 && c->corr_radius <= max_radius,
                "%s: corr_levels=%d corr_radius=%d", name, c->corr_levels, c->corr_radius);
  if (levels_fit_grid) {
    int lh[PFB_MAX_LEVELS], lw[PFB_MAX_LEVELS];
    PFB_TRY(pfb_corr_level_sizes(c->H, c->W, c->corr_levels, pool_min_side, lh, lw) > 0 ? PFB_OK : PFB_ERR_ARG);
    PFB_CHECK_ARG(lh[c->corr_levels - 1] >= 1 && lw[c->corr_levels - 1] >= 1, "%s: %dx%d grid too small for %d levels", name, c->H, c->W,
                  c->corr_levels);
  }
  PFB_CHECK_ARG(c->iters >= 0, "%s: iters=%d", name, c->iters);
  PFB_CHECK_ARG(c->volume_layout == 0 || (c->volume_layout == 1 && c->dtype != PFB_F32 && !c->alternate_corr && c->corr_levels <= 4),
                "%s: volume_layout=%d needs f16/bf16, a materialised pyramid and <= 4 levels", name, c->volume_layout);
  return PFB_OK;
}

int check_loop_buffers(const pfb_raft_cfg* c, const pfb_raft_buffers* buf, bool need_pyramid, size_t need, const char* name) {
  PFB_CHECK_ARG(buf, "%s: null buffers", name);
  PFB_CHECK_ARG(buf->net && buf->inp && buf->coords && buf->workspace, "%s: null state buffer", name);
  if (need_pyramid) {
    PFB_CHECK_ARG(buf->pyramid, "%s: null pyramid", name);
    PFB_CHECK_ARG(!c->alternate_corr || (buf->fmap1 && c->feat_dim > 0), "%s: alternate_corr needs fmap1 and feat_dim", name);
  }
  PFB_CHECK_ARG(buf->pool_min_side >= 0 && (buf->pool_min_side == 0 || !c->alternate_corr),
                "%s: pool_min_side=%d (positive values describe a materialised pyramid)", name, buf->pool_min_side);
  PFB_CHECK_ARG(buf->workspace_bytes >= need, "%s: workspace %zu bytes < required %zu", name, buf->workspace_bytes, need);
  return PFB_OK;
}

int copy_wide_state(const pfb_raft_cfg* c, const pfb_raft_buffers* buf, void* X, int x_stride, bool to_wide, cudaStream_t s) {
  const size_t es = dtype_size(c->dtype), P = (size_t)c->B * c->H * c->W, row = 128 * es, pitch = x_stride * es;
  char* x = reinterpret_cast<char*>(X);
  if (!to_wide) {
    PFB_CUDA(cudaMemcpy2DAsync(buf->net, row, x, pitch, row, P, cudaMemcpyDeviceToDevice, s));
    return PFB_OK;
  }
  PFB_CUDA(cudaMemcpy2DAsync(x, pitch, buf->net, row, row, P, cudaMemcpyDeviceToDevice, s));
  PFB_CUDA(cudaMemcpy2DAsync(x + row, pitch, buf->inp, row, row, P, cudaMemcpyDeviceToDevice, s));
  return PFB_OK;
}

int raft_lookup(const pfb_raft_cfg* c, void* const* pyramid, const void* fmap1, const float* coords, void* out, int out_stride,
                void* flags, cudaStream_t s, float scale, int pool_min_side) {
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
  // RAFT's pyramid (pool_min_side = 0) keeps the lookups' own H >> l sizes; a pyramid that stops pooling passes them explicitly
  int lh[PFB_MAX_LEVELS], lw[PFB_MAX_LEVELS];
  const bool sized = pool_min_side > 0;
  if (sized && pfb_corr_level_sizes(c->H, c->W, c->corr_levels, pool_min_side, lh, lw) < 1) return PFB_ERR_ARG;
  if (c->volume_layout == 1)
    return pfb_corr_lookup_tiled_ex(pyramid, sized ? lh : nullptr, sized ? lw : nullptr, coords, out, c->B, c->H, c->W, c->H, c->W,
                                    c->corr_levels, c->corr_radius, c->dtype, out_stride, (pfb_stream)s);
  return pfb_corr_lookup_ex(pyramid, sized ? lh : nullptr, sized ? lw : nullptr, coords, out, c->B, c->H, c->W, c->corr_levels,
                            c->corr_radius, c->dtype, c->dtype, 0, out_stride, (pfb_stream)s);
}

int motion_encoder(const pfb_raft_cfg* c, cudaStream_t s, const ConvExtras& e, const MotionLayers& L, const MotionBuffers& m,
                   const pfb_conv_src& corr, const ConvOut& out, cudaStream_t side, cudaEvent_t ev_join, const pfb_layer* c2f2) {
  const int c_corflo = m.c_cor2 + m.c_flo2;
  const cudaStream_t sf = side ? side : s;  // the flow branch's launches
  if (L.convc2) {
    PFB_TRY(launch_conv(c, s, *L.convc1, {corr}, {PFB_EPI_RELU, m.cor1, m.c_cor1, 0}, e));
    if (!c2f2) PFB_TRY(launch_conv(c, s, *L.convc2, {src_of(m.cor1, m.c_cor1, m.c_cor1)}, {PFB_EPI_RELU, m.corflo, c_corflo, 0}, e));
  } else {
    PFB_TRY(launch_conv(c, s, *L.convc1, {corr}, {PFB_EPI_RELU, m.corflo, c_corflo, 0}, e));
  }
  const pfb_layer& LF = *L.convf1;
  static const int env_fc = getenv("PFB_FLOW_CONV_UMMA") ? atoi(getenv("PFB_FLOW_CONV_UMMA")) : 1;
  if (env_fc && LF.weight_k && LF.KH == 7 && LF.KW == 7 && LF.Cin == 2 && LF.Cout == 128 && c->dtype != PFB_F32 && c->impl != 1)
    PFB_TRY(pfb_flow_conv7x7(e.flow, LF.weight_k, LF.bias, m.flo1, m.c_flo1, 0, c->B, c->H, c->W, c->dtype, (pfb_stream)sf));
  else
    PFB_TRY(launch_conv(c, sf, LF, {src_of(e.flow, 2, 2, 0, 1)}, {PFB_EPI_RELU, m.flo1, m.c_flo1, 0}, e));
  if (c2f2)  // [cor1 | flo1] -> [cor | flo]
    PFB_TRY(launch_conv(c, s, *c2f2, {src_of(m.cor1, m.c_cor1, m.c_cor1), src_of(m.flo1, m.c_flo1, m.c_flo1)},
                        {PFB_EPI_RELU, m.corflo, c_corflo, 0}, e));
  else
    PFB_TRY(launch_conv(c, sf, *L.convf2, {src_of(m.flo1, m.c_flo1, m.c_flo1)}, {PFB_EPI_RELU, m.corflo, c_corflo, m.c_cor2}, e));
  if (side) {  // join: `conv` reads both branches
    PFB_CUDA(cudaEventRecord(ev_join, side));
    PFB_CUDA(cudaStreamWaitEvent(s, ev_join, 0));
  }
  return launch_conv(c, s, *L.conv, {src_of(m.corflo, c_corflo, c_corflo)}, out, e);
}

int flow_head(const pfb_raft_cfg* c, cudaStream_t s, const ConvExtras& e, const pfb_layer& flow1, const pfb_layer& flow2,
              const pfb_layer* flow2t, const pfb_conv_src& net, void* fh, int c_fh, float* taps, float* flow) {
  PFB_TRY(launch_conv(c, s, flow1, {net}, {PFB_EPI_RELU, fh, c_fh, 0}, e));
  if (flow2t && flow2t->weight_k && c->dtype != PFB_F32 && c->impl != 1) {
    PFB_TRY(launch_conv(c, s, *flow2t, {src_of(fh, c_fh, c_fh)}, {PFB_EPI_LINEAR_F32, taps, 32, 0}, e));
    return pfb_flow_tap_gather(taps, 32, flow2.bias, e.coords, flow, c->B, c->H, c->W, (pfb_stream)s);
  }
  return launch_conv(c, s, flow2, {src_of(fh, c_fh, c_fh)}, {PFB_EPI_FLOW, flow, 2, 0}, e);
}

int mask_head(const pfb_raft_cfg* c, cudaStream_t s, const ConvExtras& e, const pfb_layer& mask1, const pfb_layer& mask2,
              const pfb_conv_src& net, void* mh, void* mask, int channels) {
  PFB_TRY(launch_conv(c, s, mask1, {net}, {PFB_EPI_RELU, mh, 256, 0}, e));
  return launch_conv(c, s, mask2, {src_of(mh, 256, 256)}, {PFB_EPI_LINEAR, mask, channels, 0, 0.25f}, e);
}

static int heads_of(const pfb_raft_cfg* c) { return c->num_heads > 0 ? c->num_heads : 1; }

int gma_aggregate(const pfb_raft_cfg* c, const pfb_layer& agg_v, const pfb_layer& agg_proj, const void* attention_ptr, float gamma,
                  void* motion, int motion_stride, int motion_offset, int out_offset, void* vbuf_ptr, void* vT_ptr, void* agg_ptr, int n_pad,
                  cudaStream_t s, const float* mode_score) {
  PFB_CHECK_ARG(attention_ptr, "gma: null attention");
  const int N = c->H * c->W, heads = heads_of(c), vdim = heads * 128;
  const size_t es = dtype_size(c->dtype);
  const char* attention = reinterpret_cast<const char*>(attention_ptr);
  char* vbuf = reinterpret_cast<char*>(vbuf_ptr);
  char* vT = reinterpret_cast<char*>(vT_ptr);
  // one head: attn @ v goes straight into the AXPY epilogue.  Several heads (gma_utils.py:101-111): every head's attn @ v
  // lands in its 128 columns of `agg`, then project (heads*128 -> 128) carries the AXPY epilogue.
  char* agg = heads > 1 ? reinterpret_cast<char*>(agg_ptr) : nullptr;
  // CRAFT (mode_score): the heads are the aggregator's modes, and pfb_craft_mode_aggregate of [motion | the heads' attn @ v] replaces
  // project + AXPY (setrans.py:423-471); one mode's attn @ v lands in the motion_global columns and is aggregated there in place
  PFB_CHECK_ARG(heads == 1 || mode_score || (agg_proj.weight && agg_proj.Cin == vdim),
                "gma: num_heads=%d needs the Aggregate.project layer (%d -> 128)", heads, vdim);
  PFB_CHECK_ARG(agg_v.weight && agg_v.Cin == 128, "gma: Aggregate.to_v layer missing");
  {  // v = to_v(motion)
    ConvExtras e;
    e.hidden = c->hidden_dim;
    PFB_TRY(launch_conv(c, s, agg_v, {src_of(motion, 128, motion_stride, motion_offset)}, {PFB_EPI_LINEAR, vbuf, vdim, 0}, e));
  }
  const bool tensor_path = c->dtype != PFB_F32 && c->impl != 1 && (N % 8) == 0;
  if (tensor_path) PFB_TRY(pfb_transpose_pm(vbuf, vT, c->B, N, vdim, n_pad, c->dtype, (pfb_stream)s));
  static const int env_batched = getenv("PFB_GMA_BATCHED") ? atoi(getenv("PFB_GMA_BATCHED")) : 1;
  // "1x1 convolution" of head h over sample b (b < 0: all samples in one launch): pixels = queries, input channels = the N
  // attention columns, weights = the sample's v (SIMT layout [N][vdim], columns h*128...) / v^T (K-major [vdim][n_pad], rows
  // h*128...).  The attention is head-major, so every operand is affine in the pixel index.
  auto attn_v = [&](int h, int b) -> int {
    const int b0 = b < 0 ? 0 : b;
    const pfb_layer v{vbuf + ((size_t)b0 * N * vdim + (size_t)h * 128) * es, nullptr, 128, vdim, N, 1, 1,
                      tensor_path ? vT + ((size_t)b0 * vdim + (size_t)h * 128) * n_pad * es : nullptr, tensor_path ? n_pad : 0,
                      tensor_path ? 128 : 0};
    ConvExtras e;
    e.B = b < 0 ? 0 : 1;
    if (b < 0) {
      // ONE launch for all samples: per-sample weights = that sample's v^T (rows b * vdim + h * 128 ...).  B x 55 row tiles
      // fill the machine; one launch per sample left only 55 row tiles, a fraction of the machine.
      e.impl = 2;
      e.w_rows_per_sample = vdim;
    }
    const pfb_conv_src a = src_of(attention + ((size_t)h * c->B + b0) * N * N * es, N, N);
    if (heads > 1) return launch_conv(c, s, v, {a}, {PFB_EPI_LINEAR, agg + (size_t)b0 * N * vdim * es, vdim, h * 128}, e);
    char* mrow = reinterpret_cast<char*>(motion) + (size_t)b0 * N * motion_stride * es;
    if (mode_score) return launch_conv(c, s, v, {a}, {PFB_EPI_LINEAR, mrow, motion_stride, out_offset}, e);
    e.aux_h = mrow + (size_t)motion_offset * es;
    e.hidden = motion_stride;
    return launch_conv(c, s, v, {a}, {PFB_EPI_AXPY, mrow, motion_stride, out_offset, gamma}, e);
  };
  for (int h = 0; h < heads; ++h) {
    if (tensor_path && env_batched) PFB_TRY(attn_v(h, -1));
    else for (int b = 0; b < c->B; ++b) PFB_TRY(attn_v(h, b));
  }
  if (mode_score) {
    const int P = c->B * N;
    return heads > 1 ? pfb_craft_mode_aggregate(agg, vdim, heads, 128, mode_score, gamma, motion, motion_stride, motion_offset, motion,
                                                motion_stride, out_offset, P, c->dtype, (pfb_stream)s)
                     : pfb_craft_mode_aggregate(reinterpret_cast<char*>(motion) + (size_t)out_offset * es, motion_stride, 1, 128, mode_score,
                                                gamma, motion, motion_stride, motion_offset, motion, motion_stride, out_offset, P, c->dtype,
                                                (pfb_stream)s);
  }
  if (heads > 1) {  // motion_global = motion + gamma * project(out)   gma_utils.py:108-111
    pfb_layer proj = agg_proj;
    proj.bias = nullptr;  // Aggregate.project has no bias
    ConvExtras e;
    e.aux_h = reinterpret_cast<char*>(motion) + (size_t)motion_offset * es;
    e.hidden = motion_stride;
    PFB_TRY(launch_conv(c, s, proj, {src_of(agg, vdim, vdim)}, {PFB_EPI_AXPY, motion, motion_stride, out_offset, gamma}, e));
  }
  return PFB_OK;
}

int check_multiscale_args(const pfb_raft_cfg* c, const pfb_raft_buffers* buf, float corr_scale, const float* next_coords, int upflow2,
                          const char* name) {
  PFB_CHECK_ARG(c->iters >= 1, "%s: every scale needs at least one iteration (iters=%d)", name, c->iters);
  PFB_CHECK_ARG(corr_scale >= 0.f, "%s: corr_scale=%g", name, (double)corr_scale);
  PFB_CHECK_ARG(next_coords || buf->flow_up, "%s: needs next_coords (coarser scales) or flow_up (the finest)", name);
  if (next_coords) return PFB_OK;
  const int f = 2 << upflow2;  // the output grid is f times this scale's
  PFB_CHECK_ARG(c->out_h > 0 && c->out_w > 0 && c->pad_top >= 0 && c->pad_left >= 0 && c->out_h + c->pad_top <= f * c->H &&
                    c->out_w + c->pad_left <= f * c->W,
                "%s: output window %dx%d+(%d,%d) outside %dx%d", name, c->out_h, c->out_w, c->pad_top, c->pad_left, f * c->H, f * c->W);
  PFB_CHECK_ARG(!buf->flow_small || (c->out_h >= 16 && c->out_w >= 16), "%s: output %dx%d smaller than 16 px per side", name, c->out_h,
                c->out_w);
  return PFB_OK;
}

// ---- the raft / raft_small / gma / ms_raft_plus / ccmr / flow1d / csflow / scv loop ----

enum LoopFamily { FAMILY_RAFT, FAMILY_MSRAFT, FAMILY_CCMR };  // the pfb_raft_*, pfb_msraft_* or pfb_ccmr_* entry points
static const char* const kFamilyName[] = {"raft", "msraft", "ccmr"};
enum LookupKind { LOOKUP_PYRAMID, LOOKUP_1D, LOOKUP_STRIP, LOOKUP_SPARSE };  // RAFT's, flow1d's rows / columns, csflow's strips, scv's k-NN
enum Aggregate { AGG_NONE, AGG_GMA, AGG_CCMR };  // motion_global beside motion (a 256-channel motion buffer), and by what
struct LoopSpec {
  LoopFamily family; LookupKind lookup; Aggregate aggregate;
  bool small;    // SmallUpdateBlock: 96 / 64 widths, one ConvGRU half, no context terms, flow2t or mask head, SIMT only
  int upsample;  // the convex upsample's factor (mask of 9 taps x upsample^2 channels); 0: no mask, pfb_raft_refine ends in upflow8
};
// What a variant's loop is made of (every per-model decision of this file reads it); null for the variants this loop does not run
static const LoopSpec* loop_spec(int variant) {
  static const LoopSpec raft{FAMILY_RAFT, LOOKUP_PYRAMID, AGG_NONE, false, 8}, raft_small{FAMILY_RAFT, LOOKUP_PYRAMID, AGG_NONE, true, 0},
      gma{FAMILY_RAFT, LOOKUP_PYRAMID, AGG_GMA, false, 8}, ms_raft_p{FAMILY_MSRAFT, LOOKUP_PYRAMID, AGG_NONE, false, 2},
      ccmr{FAMILY_CCMR, LOOKUP_PYRAMID, AGG_CCMR, false, 2}, flow1d{FAMILY_RAFT, LOOKUP_1D, AGG_NONE, false, 8},
      csflow{FAMILY_RAFT, LOOKUP_STRIP, AGG_NONE, false, 8}, scv8{FAMILY_RAFT, LOOKUP_SPARSE, AGG_NONE, false, 8},
      scv4{FAMILY_RAFT, LOOKUP_SPARSE, AGG_NONE, false, 4};
  static const LoopSpec* const by_variant[PFB_VARIANT_COUNT] = {  // in pfb_variant order
      &raft, &raft_small, &gma, nullptr /* skflow */, nullptr /* sea_raft */, &ms_raft_p, &ccmr, &flow1d, &csflow, &scv8, &scv4};
  return (unsigned)variant < PFB_VARIANT_COUNT ? by_variant[variant] : nullptr;
}
static int mask_channels(const LoopSpec& sp) { return 9 * sp.upsample * sp.upsample; }

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

// of a cfg check_cfg accepted
static Workspace plan(const pfb_raft_cfg* c) {
  const LoopSpec& sp = *loop_spec(c->variant);
  Workspace w{};
  const size_t vdim = (size_t)heads_of(c) * 128;
  const size_t P = (size_t)c->B * c->H * c->W;
  const size_t es = dtype_size(c->dtype);
  const int K = 2 * c->corr_radius + 1;
  // flow1d: [corr_x taps | corr_y taps]; csflow: [4D taps of every level | strip taps of every level]
  w.planes = sp.lookup == LOOKUP_1D ? 2 * K : (sp.lookup == LOOKUP_STRIP ? 2 : 1) * c->corr_levels * K * K;
  // 16-byte aligned rows for the tensor-core path (the TMA unit zero-fills a partial last 64-channel K chunk itself)
  w.corr_stride = (c->dtype == PFB_F32) ? w.planes : (int)align_up(w.planes, 8);
  if (!sp.small) {
    w.c_cor1 = 256; w.c_cor2 = 192; w.c_flo1 = 128; w.c_flo2 = 64; w.c_fh = 256;
    // gma and ccmr keep [motion | motion_global] side by side so the GRU still sees three sources (update.py:150-151)
    w.c_motion = sp.aggregate != AGG_NONE ? 256 : 128;
  } else {
    w.c_cor1 = 0; w.c_cor2 = 96; w.c_flo1 = 64; w.c_flo2 = 32; w.c_motion = 82; w.c_fh = 128;
  }
  w.c_corflo = w.c_cor2 + w.c_flo2;
  Carve k;
  w.off_corr = k.take(P * w.corr_stride * es);
  w.off_cor1 = k.take(P * (size_t)w.c_cor1 * es);
  w.off_corflo = k.take(P * (size_t)w.c_corflo * es);
  w.off_flo1 = k.take(P * (size_t)w.c_flo1 * es);
  w.off_motion = k.take(P * (size_t)w.c_motion * es);
  w.off_z = k.take(P * (size_t)c->hidden_dim * es);
  w.off_rh = k.take(P * (size_t)c->hidden_dim * es);
  w.off_fh = k.take(P * (size_t)w.c_fh * es);
  w.off_mh = k.take(sp.upsample ? P * 256 * es : 0);
  w.off_mask = k.take(P * (size_t)mask_channels(sp) * es);
  w.off_flow = k.take(P * 2 * sizeof(float));
  w.off_taps = k.take(!sp.small ? P * 32 * sizeof(float) : 0);
  w.n_pad = (int)align_up((size_t)c->H * c->W, 64);
  w.off_vbuf = k.take(sp.aggregate == AGG_GMA ? P * vdim * es : 0);
  w.off_vT = k.take(sp.aggregate == AGG_GMA ? (size_t)c->B * vdim * w.n_pad * es : 0);
  w.off_agg = k.take(sp.aggregate == AGG_GMA && vdim > 128 ? P * vdim * es : 0);
  w.off_flags = k.take(c->alternate_corr ? P : 0);
  for (int i = 0; i < 4; ++i)
    w.off_ctx[i] = k.take((!sp.small && c->dtype != PFB_F32) ? P * (size_t)((i & 1) ? c->hidden_dim : 2 * c->hidden_dim) * es : 0);
  w.total = k.total;
  return w;
}

// buf: the buffers of a run (or of pfb_raft_workspace_bytes_ex), whose pool_min_side sizes the pyramid levels that must not be empty;
// NULL checks them as RAFT's pyramid sizes them
static int check_cfg(const pfb_raft_cfg* c, LoopFamily family, const pfb_raft_buffers* buf = nullptr) {
  const char* name = kFamilyName[family];
  PFB_CHECK_ARG(c, "%s: null cfg", name);
  const LoopSpec* sp = loop_spec(c->variant);
  PFB_CHECK_ARG(sp && sp->family == family, "%s: variant=%d is not a loop of the pfb_%s_* entry points", name, c->variant, name);
  const int pool_min_side = buf && buf->pool_min_side > 0 ? buf->pool_min_side : 0;
  PFB_TRY(check_loop_cfg(c, name, sp->lookup != LOOKUP_SPARSE, sp->lookup == LOOKUP_1D ? 64 : 15, pool_min_side));
  switch (sp->lookup) {
    case LOOKUP_SPARSE:  // 5 levels of 9 x 9 bins (scv.py:245-260) over a table of feat_dim = num_k matches per query
      PFB_CHECK_ARG(c->corr_levels == 5 && c->corr_radius == 4 && !c->alternate_corr && c->volume_layout == 0 && c->feat_dim >= 1 &&
                        c->feat_dim <= 32 && c->feat_dim <= c->H * c->W,
                    "scv: needs corr_levels=5, corr_radius=4, the sparse table (volume_layout=0) and num_k (feat_dim) in 1..min(32, H*W) "
                    "(got levels=%d radius=%d alternate_corr=%d volume_layout=%d num_k=%d grid %dx%d)", c->corr_levels, c->corr_radius,
                    c->alternate_corr, c->volume_layout, c->feat_dim, c->H, c->W); break;
    case LOOKUP_STRIP:  // the reference's pyramid always has 4 levels (csflow.py:158, 448) and its strips need a materialised volume
      PFB_CHECK_ARG(c->corr_levels == 4 && !c->alternate_corr && (c->volume_layout == 0 || c->volume_layout == 1),
                    "csflow: needs corr_levels=4 and a materialised dense or tiled volume (got levels=%d alternate_corr=%d volume_layout=%d)",
                    c->corr_levels, c->alternate_corr, c->volume_layout); break;
    case LOOKUP_1D:  // two 1D volumes, looked up along rows / columns of at least two pixels (flow1d/correlation.py:41, 66)
      PFB_CHECK_ARG(c->corr_levels == 1 && c->corr_radius >= 1 && !c->alternate_corr && c->volume_layout == 0 && c->H >= 2 && c->W >= 2,
                    "flow1d: needs corr_levels=1, corr_radius 1..64, a materialised dense volume and a grid of at least 2x2 (got levels=%d "
                    "radius=%d alternate_corr=%d volume_layout=%d grid %dx%d)", c->corr_levels, c->corr_radius, c->alternate_corr,
                    c->volume_layout, c->H, c->W); break;
    case LOOKUP_PYRAMID: break;
  }
  PFB_CHECK_ARG(c->num_heads >= 0 && c->num_heads <= 64 && (sp->aggregate == AGG_GMA || heads_of(c) == 1), "%s: num_heads=%d", name, c->num_heads);
  // gma also takes a 256-channel static GRU input: SplatFlow's [inp | mf_t] (a24); the context split handles any context width
  if (!sp->small)
    PFB_CHECK_ARG(c->hidden_dim == 128 && (c->context_dim == 128 || (c->variant == PFB_VARIANT_GMA && c->context_dim == 256)),
                  "%s: the update block expects hidden=context=128 (gma: context 128 or 256)", name);
  else PFB_CHECK_ARG(c->hidden_dim == 96 && c->context_dim == 64, "raft_small: SmallUpdateBlock expects hidden=96 context=64");
  return PFB_OK;
}

struct Ctx {
  const pfb_raft_cfg* c;
  const LoopSpec* sp;
  const pfb_raft_weights* w;
  const pfb_raft_buffers* b;
  Workspace ws;
  char* base;
  cudaStream_t s;
  ConvExtras e;            // every layer's GRU operands, coordinates and flow
  float corr_scale = 0.f;  // on-the-fly lookup scale (0: 1/sqrt(feat_dim))
  const pfb_ccmr_weights* ccmr = nullptr;  // ccmr: the XCiT blocks of the scale, and their part of the workspace
  char* ccmr_base = nullptr;
  // flow branch of the motion encoder on a second stream (fork_flow_branch): null when not forked
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  void* at(size_t off) const { return base + off; }
};

static int run_conv(const Ctx& x, int layer, std::initializer_list<pfb_conv_src> srcs, const ConvOut& o, const void* addend = nullptr,
                    int addend_stride = 0) {
  ConvExtras e = x.e;
  e.addend = addend; e.addend_stride = addend_stride;
  return launch_conv(x.c, x.s, x.w->layers[layer], srcs, o, e);
}

// round-2 restructurings of the tensor-core path; PFB_GRU_CTX_SPLIT=0 / PFB_MERGE_C2F2=0 fall back to the plain layers
static bool tensor_path(const Ctx& x) { return !x.sp->small && x.c->dtype != PFB_F32 && x.c->impl != 1; }
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
    PFB_TRY(run_conv(x, layers[i], {src_of(x.b->inp, cd, cd)}, {PFB_EPI_LINEAR, x.at(x.ws.off_ctx[i]), n, 0}));
  }
  return PFB_OK;
}

static int lookup(const Ctx& x) {
  if (x.sp->lookup == LOOKUP_SPARSE)
    return pfb_sparse_lookup(reinterpret_cast<const float*>(x.b->pyramid[0]), x.b->coords, x.at(x.ws.off_corr), x.c->B, x.c->H, x.c->W,
                             x.c->feat_dim, x.c->dtype, x.ws.corr_stride, (pfb_stream)x.s);
  if (x.sp->lookup == LOOKUP_1D)
    return pfb_corr1d_lookup(x.b->pyramid[0], x.b->pyramid[1], x.b->coords, x.at(x.ws.off_corr), x.c->B, x.c->H, x.c->W, x.c->corr_radius,
                             x.c->dtype, x.ws.corr_stride, (pfb_stream)x.s);
  PFB_TRY(raft_lookup(x.c, x.b->pyramid, x.b->fmap1, x.b->coords, x.at(x.ws.off_corr), x.ws.corr_stride, x.at(x.ws.off_flags), x.s,
                      x.corr_scale, x.b->pool_min_side));
  if (x.sp->lookup != LOOKUP_STRIP) return PFB_OK;
  // csflow: the 4D lookup above wrote planes 0 .. L K^2 - 1 and zero-filled the rest; the strip taps follow (a20)
  const int L = x.c->corr_levels, K = 2 * x.c->corr_radius + 1;
  return pfb_strip_lookup(reinterpret_cast<const float*>(x.b->pyramid[L]), reinterpret_cast<const float*>(x.b->pyramid[L + 1]),
                          x.b->coords, x.at(x.ws.off_corr), x.c->B, x.c->H, x.c->W, L, x.c->corr_radius, x.c->dtype, x.ws.corr_stride,
                          L * K * K, (pfb_stream)x.s);
}

// One BasicUpdateBlock / SmallUpdateBlock evaluation + coords update.  update.py:122-153
static int update_iter(const Ctx& x, const void* corr_ext, void* mask_out) {
  const pfb_raft_cfg* c = x.c;
  const LoopSpec& sp = *x.sp;
  const Workspace& ws = x.ws;
  const pfb_layer* L = x.w->layers;
  const int hd = c->hidden_dim, cd = c->context_dim;
  const void* corr = corr_ext ? corr_ext : x.at(ws.off_corr);
  const int corr_stride = corr_ext ? ws.planes : ws.corr_stride;
  void* motion = x.at(ws.off_motion);
  void* rh = x.at(ws.off_rh);
  const pfb_conv_src net = src_of(x.b->net, hd, hd);

  // ---- motion encoder (update.py:76-112); when forked, the fork itself is in the caller, before the lookup ----
  const MotionLayers ml{&L[PFB_L_CONVC1], !sp.small ? &L[PFB_L_CONVC2] : nullptr, &L[PFB_L_CONVF1], &L[PFB_L_CONVF2], &L[PFB_L_CONV]};
  const MotionBuffers mb{x.at(ws.off_cor1), x.at(ws.off_corflo), x.at(ws.off_flo1), ws.c_cor1, ws.c_cor2, ws.c_flo1, ws.c_flo2};
  PFB_TRY(motion_encoder(c, x.s, x.e, ml, mb, src_of(corr, ws.planes, corr_stride), {PFB_EPI_RELU_APPEND_FLOW, motion, ws.c_motion, 0},
                         x.side, x.ev_join, merged_c2f2_active(x) ? &L[PFB_L_CONVC2F2] : nullptr));

  // ---- gma: motion_global = motion + gamma * (attention @ to_v(motion))   gma_utils.py:101-113, gma/update.py:149 ----
  if (sp.aggregate == AGG_GMA)
    PFB_TRY(gma_aggregate(c, L[PFB_L_AGG_V], L[PFB_L_AGG_PROJ], x.b->attention, x.b->agg_gamma, motion, ws.c_motion, 0, 128,
                          x.at(ws.off_vbuf), x.at(ws.off_vT), x.at(ws.off_agg), ws.n_pad, x.s, x.b->agg_score));
  // ---- ccmr: motion_global = aggregator(global_context, motion)   ccmr/update.py:156-161 ----
  if (sp.aggregate == AGG_CCMR) PFB_TRY(ccmr_aggregate(c, x.ccmr, motion, ws.c_motion, x.ccmr_base, x.s));

  // ---- GRU (update.py:24-32 ConvGRU, :58-73 SepConvGRU); x = [inp, motion (, motion_global)] ----
  const int halves = sp.small ? 1 : 2;
  const bool split = ctx_split_active(x);
  const pfb_conv_src mot = src_of(motion, ws.c_motion, ws.c_motion), hr = src_of(rh, hd, hd);
  for (int h = 0; h < halves; ++h) {
    if (split) {
      // conv([h | inp | motion]) = conv_inp(inp) + bias (once per forward, run_context_terms) + conv_rest([h | motion]) (here)
      const int lzr = h == 0 ? PFB_L_GRUX_ZR1 : PFB_L_GRUX_ZR2, lq = h == 0 ? PFB_L_GRUX_Q1 : PFB_L_GRUX_Q2;
      PFB_TRY(run_conv(x, lzr, {net, mot}, {PFB_EPI_GRU_ZR, rh, hd, 0}, x.at(ws.off_ctx[2 * h]), 2 * hd));
      PFB_TRY(run_conv(x, lq, {hr, mot}, {PFB_EPI_GRU_Q, x.b->net, hd, 0}, x.at(ws.off_ctx[2 * h + 1]), hd));
      continue;
    }
    const int lzr = h == 0 ? PFB_L_GRU_ZR1 : PFB_L_GRU_ZR2, lq = h == 0 ? PFB_L_GRU_Q1 : PFB_L_GRU_Q2;
    const pfb_conv_src inp = src_of(x.b->inp, cd, cd);
    PFB_TRY(run_conv(x, lzr, {net, inp, mot}, {PFB_EPI_GRU_ZR, rh, hd, 0}));
    PFB_TRY(run_conv(x, lq, {hr, inp, mot}, {PFB_EPI_GRU_Q, x.b->net, hd, 0}));
  }

  // ---- heads (update.py:6-14, :138-152) ----
  const bool mask = mask_out && sp.upsample;
  const bool fork_mask = x.side && mask;
  if (fork_mask) {  // last iteration: the mask head beside the flow head (both read the final hidden state)
    PFB_CUDA(cudaEventRecord(x.ev_fork, x.s));
    PFB_CUDA(cudaStreamWaitEvent(x.side, x.ev_fork, 0));
    PFB_TRY(mask_head(c, x.side, x.e, L[PFB_L_MASK1], L[PFB_L_MASK2], net, x.at(ws.off_mh), mask_out, mask_channels(sp)));
    PFB_CUDA(cudaEventRecord(x.ev_join, x.side));
  }
  PFB_TRY(flow_head(c, x.s, x.e, L[PFB_L_FLOW1], L[PFB_L_FLOW2], !sp.small ? &L[PFB_L_FLOW2T] : nullptr, net, x.at(ws.off_fh),
                    ws.c_fh, reinterpret_cast<float*>(x.at(ws.off_taps)), reinterpret_cast<float*>(x.at(ws.off_flow))));
  if (fork_mask) PFB_CUDA(cudaStreamWaitEvent(x.s, x.ev_join, 0));  // the upsample reads the mask
  else if (mask) PFB_TRY(mask_head(c, x.s, x.e, L[PFB_L_MASK1], L[PFB_L_MASK2], net, x.at(ws.off_mh), mask_out, mask_channels(sp)));
  return PFB_OK;
}

static int make_ctx(Ctx& x, const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                    cudaStream_t s, bool need_pyramid, LoopFamily family) {
  PFB_TRY(check_cfg(cfg, family, buf));
  const char* name = kFamilyName[family];
  PFB_CHECK_ARG(w, "%s: null weights", name);
  x.c = cfg; x.sp = loop_spec(cfg->variant); x.w = w; x.b = buf; x.s = s;
  x.ws = plan(cfg);
  PFB_TRY(check_loop_buffers(cfg, buf, need_pyramid, x.ws.total + (family == FAMILY_CCMR ? ccmr_plan(cfg).total : 0), name));
  x.base = reinterpret_cast<char*>(buf->workspace);
  x.e.aux_h = buf->net; x.e.aux_z = x.at(x.ws.off_z); x.e.hidden = cfg->hidden_dim;
  x.e.coords = buf->coords; x.e.flow = reinterpret_cast<const float*>(x.at(x.ws.off_flow));
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

// the workspace of the msraft / ccmr / raft entry points (ccmr's holds its XCiT plan after the loop's); 0 for a cfg they refuse
static size_t workspace_bytes(const pfb_raft_cfg* cfg, LoopFamily family, const pfb_raft_buffers* buf = nullptr) {
  if (check_cfg(cfg, family, buf) != PFB_OK) return 0;
  return plan(cfg).total + (family == FAMILY_CCMR ? ccmr_plan(cfg).total : 0);
}

// one update-block evaluation from the entry coordinates, on a built context: the flow, the context terms, the lookup unless the
// caller hands in the correlation
static int update_iter_once(Ctx& x, const void* corr, void* mask_out) {
  PFB_TRY(launch_flow_from_coords(x.b->coords, reinterpret_cast<float*>(x.at(x.ws.off_flow)), x.c->B, x.c->H, x.c->W, x.s));
  PFB_TRY(run_context_terms(x));
  if (!corr) PFB_TRY(lookup(x));
  return update_iter(x, corr, mask_out);
}

extern "C" PFB_API size_t pfb_raft_workspace_bytes(const pfb_raft_cfg* cfg) { return workspace_bytes(cfg, FAMILY_RAFT); }

extern "C" PFB_API size_t pfb_raft_workspace_bytes_ex(const pfb_raft_cfg* cfg, int pool_min_side) {
  if (pool_min_side < 0) return 0;
  pfb_raft_buffers buf{};
  buf.pool_min_side = pool_min_side;
  return workspace_bytes(cfg, FAMILY_RAFT, &buf);
}

extern "C" PFB_API int pfb_raft_workspace_motion(const pfb_raft_cfg* cfg, size_t* offset, int* channel_stride) {
  PFB_CHECK_ARG(offset && channel_stride, "raft_workspace_motion: null output");
  PFB_TRY(check_cfg(cfg, FAMILY_RAFT));
  const Workspace w = plan(cfg);
  *offset = w.off_motion;
  *channel_stride = w.c_motion;
  return PFB_OK;
}

extern "C" PFB_API int pfb_raft_update_iter(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                                    const void* corr, void* mask_out, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr, FAMILY_RAFT));
  return update_iter_once(x, corr, mask_out);
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
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), true, FAMILY_RAFT));
  PFB_CHECK_ARG(buf->flow_up, "raft_refine: null flow_up");
  PFB_CHECK_ARG(!x.sp->upsample || cfg->iters >= 1, "raft_refine: the convex upsample needs at least one iteration (mask)");
  void* mask = x.sp->upsample ? x.at(x.ws.off_mask) : nullptr;
  PFB_TRY(run_iterations(x, mask));
  if (x.sp->upsample == 4)
    return pfb_convex_upsample4x(buf->coords, mask, buf->flow_up, buf->flow_small, cfg->B, cfg->H, cfg->W, cfg->out_h, cfg->out_w,
                                 cfg->pad_top, cfg->pad_left, cfg->dtype, stream);
  if (x.sp->upsample == 8)
    return pfb_convex_upsample(buf->coords, mask, buf->flow_up, buf->flow_small, cfg->B, cfg->H, cfg->W, cfg->out_h,
                               cfg->out_w, cfg->pad_top, cfg->pad_left, cfg->dtype, stream);
  return pfb_upflow8(buf->coords, buf->flow_up, buf->flow_small, cfg->B, cfg->H, cfg->W, cfg->out_h, cfg->out_w,
                     cfg->pad_top, cfg->pad_left, stream);
}

// ---- a17: MS-RAFT+ (one call per scale of ms_raft_plus.py:177-214) ----
extern "C" PFB_API size_t pfb_msraft_workspace_bytes(const pfb_raft_cfg* cfg) { return workspace_bytes(cfg, FAMILY_MSRAFT); }

extern "C" PFB_API int pfb_msraft_update_iter(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                                              const void* corr, void* mask_out, float corr_scale, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr, FAMILY_MSRAFT));
  PFB_CHECK_ARG(corr_scale >= 0.f, "msraft_update_iter: corr_scale=%g", (double)corr_scale);
  x.corr_scale = corr_scale;
  return update_iter_once(x, corr, mask_out);
}

extern "C" PFB_API int pfb_msraft_refine(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf, float corr_scale,
                                         float* next_coords, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ctx(x, cfg, w, buf, as_stream(stream), true, FAMILY_MSRAFT));
  PFB_TRY(check_multiscale_args(cfg, buf, corr_scale, next_coords, 0, "msraft_refine"));
  x.corr_scale = corr_scale;
  void* mask = x.at(x.ws.off_mask);
  PFB_TRY(run_iterations(x, mask));
  if (next_coords)  // handover: the absolute coordinates, doubled and convex-upsampled with zero-padded taps (ms_raft_plus.py:198-200)
    return pfb_convex_upsample2x(buf->coords, mask, next_coords, 1, cfg->B, cfg->H, cfg->W, 0, 0, 0, 0, cfg->dtype, stream);
  // flow_small = downflow(flow_up, 1/16) at int(h / 16) x int(w / 16) of the un-padded size (ms_raft_plus.py:22-35, 221-224)
  return ccmr_output(cfg, buf->coords, mask, buf->flow_up, buf->flow_small, 0, nullptr, x.s);
}

// ---- a18: CCMR / CCMR+ (one call per scale of ccmr.py:179-220) ----
extern "C" PFB_API size_t pfb_ccmr_workspace_bytes(const pfb_raft_cfg* cfg) { return workspace_bytes(cfg, FAMILY_CCMR); }

static int make_ccmr_ctx(Ctx& x, const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf, cudaStream_t s,
                         bool need_pyramid, float corr_scale) {
  PFB_CHECK_ARG(w, "ccmr: null weights");
  PFB_TRY(make_ctx(x, cfg, &w->raft, buf, s, need_pyramid, FAMILY_CCMR));
  PFB_CHECK_ARG(cfg->context_dim == 128, "ccmr: the XCiT blocks expect 128 context channels");
  x.corr_scale = corr_scale;
  x.ccmr = w;
  x.ccmr_base = x.base + x.ws.total;
  return PFB_OK;
}

extern "C" PFB_API int pfb_xcit_context(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const void* inp, void* out, void* workspace,
                                        size_t workspace_bytes, pfb_stream stream) {
  PFB_CHECK_ARG(cfg && w && inp && out && workspace, "xcit_context: null pointer");
  PFB_TRY(check_cfg(cfg, FAMILY_CCMR));
  const size_t off = plan(cfg).total, need = off + ccmr_plan(cfg).total;
  PFB_CHECK_ARG(workspace_bytes >= need, "xcit_context: workspace %zu bytes < required %zu", workspace_bytes, need);
  return ccmr_scale_setup(cfg, w, inp, out, false, reinterpret_cast<char*>(workspace) + off, as_stream(stream));
}

extern "C" PFB_API int pfb_ccmr_update_iter(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf,
                                            const void* corr, void* mask_out, float corr_scale, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ccmr_ctx(x, cfg, w, buf, as_stream(stream), corr == nullptr, corr_scale));
  PFB_CHECK_ARG(corr_scale >= 0.f, "ccmr_update_iter: corr_scale=%g", (double)corr_scale);
  PFB_TRY(ccmr_scale_setup(cfg, w, buf->inp, nullptr, true, x.ccmr_base, x.s));
  return update_iter_once(x, corr, mask_out);
}

extern "C" PFB_API int pfb_ccmr_refine(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf, float corr_scale,
                                       int upflow2, float* next_coords, pfb_stream stream) {
  Ctx x;
  PFB_TRY(make_ccmr_ctx(x, cfg, w, buf, as_stream(stream), true, corr_scale));
  PFB_CHECK_ARG(upflow2 == 0 || upflow2 == 1, "ccmr_refine: upflow2=%d (0 or 1)", upflow2);
  PFB_TRY(check_multiscale_args(cfg, buf, corr_scale, next_coords, upflow2, "ccmr_refine"));
  PFB_TRY(ccmr_scale_setup(cfg, w, buf->inp, nullptr, true, x.ccmr_base, x.s));
  void* mask = x.at(x.ws.off_mask);
  PFB_TRY(run_iterations(x, mask));
  if (next_coords)  // handover: the convex 2x of the FLOW on the next scale's grid (ccmr.py:195-202)
    return pfb_convex_handover2x(buf->coords, mask, next_coords, cfg->B, cfg->H, cfg->W, cfg->dtype, stream);
  return ccmr_output(cfg, buf->coords, mask, buf->flow_up, buf->flow_small, upflow2, x.ccmr_base, x.s);
}
