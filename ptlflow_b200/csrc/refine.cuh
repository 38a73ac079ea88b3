// Stages of the raft / gma refinement loop (refine.cu) that other loops built from the same operators reuse (skflow.cu).
#pragma once
#include "common.cuh"

namespace pfb {

// flow = coords - grid, fp32 [B,H,W,2] (misc.cu)
int launch_flow_from_coords(const float* coords, float* flow, int B, int H, int W, cudaStream_t s);

// The multi-scale lookup of the loop configured by `c` (dense, tiled or on-the-fly pyramid, as pfb_raft_refine picks it) into
// out [B,H,W,out_stride] (storage type); flags: the on-the-fly tensor-core lookup's per-query workspace (alternate_corr only).
// scale: the on-the-fly lookup's scale, 0 = 1/sqrt(feat_dim) (ms_raft_plus passes the real C when its rows carry zero channels).
int raft_lookup(const pfb_raft_cfg* c, void* const* pyramid, const void* fmap1, const float* coords, void* out, int out_stride,
                void* flags, cudaStream_t s, float scale = 0.f);

// GMA Aggregate (gma_utils.py:79-113): motion_global = motion + gamma * project(attn_h @ to_v(motion)_h), written into the
// motion buffer itself.  motion [B,H,W,motion_stride]: the motion features from channel motion_offset, motion_global to channels
// out_offset .. +127.  vbuf [P][heads*128], vT [B][heads*128][n_pad], agg (heads > 1) [P][heads*128]: scratch of the storage type.
int gma_aggregate(const pfb_raft_cfg* c, const pfb_layer& agg_v, const pfb_layer& agg_proj, const void* attention, float gamma,
                  void* motion, int motion_stride, int motion_offset, int out_offset, void* vbuf, void* vT, void* agg, int n_pad,
                  cudaStream_t s);

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
// the last scale's output: convex 2x of the flow (+ upflow2) into flow_up's window, then flow_small (may be NULL)
int ccmr_output(const pfb_raft_cfg* c, const float* coords, const void* mask, float* flow_up, float* flow_small, int upflow2, char* base,
                cudaStream_t s);

}  // namespace pfb
