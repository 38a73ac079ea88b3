// Host-side pieces of the refinement loops (refine.cu) that every loop built from the same operators shares: the convolution
// launcher, the cfg / buffer checks, the workspace carve, the lookup, RAFT's update-block stages (motion encoder, flow head, mask
// head), GMA's aggregate and the multi-scale argument check (skflow.cu, searaft.cu, ccmr.cu).
#pragma once
#include <initializer_list>

#include "common.cuh"

namespace pfb {

inline pfb_conv_src src_of(const void* ptr, int channels, int stride, int offset = 0, int is_f32 = 0) {
  pfb_conv_src s;
  s.ptr = ptr; s.channels = channels; s.stride = stride; s.offset = offset; s.is_f32 = is_f32;
  return s;
}

// Consecutive buffers of a workspace, each at a 256-byte aligned offset; `total` is the size of everything taken so far
struct Carve {
  size_t total = 0;
  size_t take(size_t bytes) {
    const size_t o = total;
    total = align_up(total + bytes, 256);
    return o;
  }
};

// Where a convolution writes: epilogue, buffer [B,H,W,stride] and first channel, and the PFB_EPI_LINEAR scale
struct ConvOut {
  int epi;
  void* ptr;
  int stride, offset;
  float scale = 1.f;
};

// The optional fields of pfb_conv_params (zero / null: not set) and two overrides of the cfg's values
struct ConvExtras {
  const void* aux_h = nullptr;  // GRU hidden state / AXPY residual, `hidden` its stride
  void* aux_z = nullptr;
  int hidden = 0;
  float* coords = nullptr;      // PFB_EPI_FLOW
  const float* flow = nullptr;  // PFB_EPI_*_APPEND_FLOW
  const void* addend = nullptr;
  int addend_stride = 0;
  const pfb_conv_src* residual = nullptr;  // PFB_EPI_RESIDUAL_GELU, with the optional post_w / post_b
  const float* post_w = nullptr;
  const float* post_b = nullptr;
  int w_rows_per_sample = 0;
  int B = 0;      // > 0: the batch instead of cfg->B (per-sample launches)
  int impl = -1;  // >= 0: the implementation instead of cfg->impl
};

// One pfb_conv2d of layer L over the concatenated sources (their channels must add up to L.Cin) on the cfg's grid and dtype
int launch_conv(const pfb_raft_cfg* c, cudaStream_t s, const pfb_layer& L, std::initializer_list<pfb_conv_src> srcs, const ConvOut& o,
                const ConvExtras& e = ConvExtras());

// The rules every loop's cfg follows (dtype, grid, levels / radius <= max_radius, volume_layout, iters >= 0); with `levels_fit_grid`
// the coarsest pyramid level (sized by pfb_corr_level_sizes with pool_min_side) must keep at least one pixel.  name: the entry point
// family, for the messages.
int check_loop_cfg(const pfb_raft_cfg* c, const char* name, bool levels_fit_grid = true, int max_radius = 15, int pool_min_side = 0);
// The state buffers, the pyramid (and fmap1 for alternate_corr) when the call looks up, and a workspace of at least `need` bytes
int check_loop_buffers(const pfb_raft_cfg* c, const pfb_raft_buffers* buf, bool need_pyramid, size_t need, const char* name);

// net -> X[:, 0:128] and inp -> X[:, 128:256] of the [P][x_stride] buffer X (to_wide), or X[:, 0:128] -> net
int copy_wide_state(const pfb_raft_cfg* c, const pfb_raft_buffers* buf, void* X, int x_stride, bool to_wide, cudaStream_t s);

// flow = coords - grid, fp32 [B,H,W,2] (misc.cu)
int launch_flow_from_coords(const float* coords, float* flow, int B, int H, int W, cudaStream_t s);

// The multi-scale lookup of the loop configured by `c` (dense, tiled or on-the-fly pyramid, as pfb_raft_refine picks it) into
// out [B,H,W,out_stride] (storage type); flags: the on-the-fly tensor-core lookup's per-query workspace (alternate_corr only).
// scale: the on-the-fly lookup's scale, 0 = 1/sqrt(feat_dim) (ms_raft_plus passes the real C when its rows carry zero channels).
// pool_min_side: pfb_raft_buffers.pool_min_side, the rule that sized the materialised pyramid's levels (pfb_corr_level_sizes).
int raft_lookup(const pfb_raft_cfg* c, void* const* pyramid, const void* fmap1, const float* coords, void* out, int out_stride,
                void* flags, cudaStream_t s, float scale = 0.f, int pool_min_side = 0);

// RAFT's motion encoder (update.py:76-112): relu(conv([relu(convc2(relu(convc1(corr)))) | relu(convf2(relu(convf1(flow))))])) and
// the flow (e.flow) into `out` (RELU_APPEND_FLOW).  convc2 == NULL: SmallMotionEncoder, convc1 writes the correlation columns of
// corflo itself.  c2f2: convc2 | convf2 as one block-diagonal layer instead of the two.  side: the stream of the flow branch
// (convf1, convf2), joined with ev_join before `conv`; NULL: everything on s.
struct MotionLayers {
  const pfb_layer *convc1, *convc2, *convf1, *convf2, *conv;
};
struct MotionBuffers {
  void *cor1, *corflo, *flo1;  // [P][c_cor1], [P][c_cor2 + c_flo2], [P][c_flo1]
  int c_cor1, c_cor2, c_flo1, c_flo2;
};
int motion_encoder(const pfb_raft_cfg* c, cudaStream_t s, const ConvExtras& e, const MotionLayers& L, const MotionBuffers& m,
                   const pfb_conv_src& corr, const ConvOut& out, cudaStream_t side = nullptr, cudaEvent_t ev_join = nullptr,
                   const pfb_layer* c2f2 = nullptr);
// RAFT's flow head (update.py:6-14): coords += flow2(relu(flow1(net))), flow = coords - grid.  With flow2t (f16 / bf16, wgmma) the
// 3x3 -> 2 convolution is one 1x1 GEMM to the 18 (tap, output) products in taps [P][32] fp32, then a 9-tap gather.
// fh: [P][c_fh] scratch.
int flow_head(const pfb_raft_cfg* c, cudaStream_t s, const ConvExtras& e, const pfb_layer& flow1, const pfb_layer& flow2,
              const pfb_layer* flow2t, const pfb_conv_src& net, void* fh, int c_fh, float* taps, float* flow);
// The convex-upsample mask 0.25 * mask2(relu(mask1(net))) (update.py:138-140) into mask [P][channels]; mh: [P][256] scratch
int mask_head(const pfb_raft_cfg* c, cudaStream_t s, const ConvExtras& e, const pfb_layer& mask1, const pfb_layer& mask2,
              const pfb_conv_src& net, void* mh, void* mask, int channels);

// GMA Aggregate (gma_utils.py:79-113): motion_global = motion + gamma * project(attn_h @ to_v(motion)_h), written into the
// motion buffer itself.  motion [B,H,W,motion_stride]: the motion features from channel motion_offset, motion_global to channels
// out_offset .. +127.  vbuf [P][heads*128], vT [B][heads*128][n_pad], agg (heads > 1) [P][heads*128]: scratch of the storage type.
int gma_aggregate(const pfb_raft_cfg* c, const pfb_layer& agg_v, const pfb_layer& agg_proj, const void* attention, float gamma,
                  void* motion, int motion_stride, int motion_offset, int out_offset, void* vbuf, void* vT, void* agg, int n_pad,
                  cudaStream_t s, const float* mode_score = nullptr);

// The arguments of one scale of ms_raft_plus / ccmr: iters >= 1, corr_scale >= 0, next_coords or flow_up, and for the last scale
// an output window inside the (2 << upflow2)-times grid and, with flow_small, at least 16 pixels per side
int check_multiscale_args(const pfb_raft_cfg* c, const pfb_raft_buffers* buf, float corr_scale, const float* next_coords, int upflow2,
                          const char* name);

// CCMR (ccmr.cu): the per-scale buffers of the XCiT blocks, placed after the update loop's workspace
struct CcmrPlan {
  size_t off_feat, off_pos_c, off_pos_a, off_x0, off_ln, off_qk, off_x1, off_t, off_u, off_gc, off_wf, off_wfk, off_bf, off_part,
      off_stats, off_gn, off_up;
  int chunks;
  size_t total;
};
CcmrPlan ccmr_plan(const pfb_raft_cfg* c);
// The scale's global context XCiT(inp) into gc_out (NULL: the plan's own buffer) and, with `aggregator`, the aggregator's residual
// stream and folded attention for the iterations.  base: the CCMR part of the workspace.
int ccmr_scale_setup(const pfb_raft_cfg* c, const pfb_ccmr_weights* w, const void* inp, void* gc_out, bool aggregator, char* base,
                     cudaStream_t s);
// motion_global = aggregator(global_context, motion) into columns 128..255 of motion [B,H,W,motion_stride] (motion in 0..127)
int ccmr_aggregate(const pfb_raft_cfg* c, const pfb_ccmr_weights* w, void* motion, int motion_stride, char* base, cudaStream_t s);
// the last scale's output of ccmr and (upflow2 = 0, base unused) ms_raft_plus: convex 2x of the flow (+ upflow2) into flow_up's
// window, then flow_small (may be NULL)
int ccmr_output(const pfb_raft_cfg* c, const float* coords, const void* mask, float* flow_up, float* flow_small, int upflow2, char* base,
                cudaStream_t s);

}  // namespace pfb
