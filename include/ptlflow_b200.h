/*
 * ptlflow_b200 -- C ABI of the H100-native (sm_90a) RAFT-family inference hot path.
 *
 * This is the drop-in boundary: a plain C interface (device pointers, sizes, a CUDA
 * stream) that replaces, for the RAFT hot path, what the reference reaches through
 *   - its native plugin `alt_cuda_corr`      ptlflow/utils/external/alt_cuda_corr/correlation.cpp:23-54
 *   - the corr-block protocol                ptlflow/models/raft/corr.py:13-118
 *   - the update block / upsampling modules  ptlflow/models/raft/update.py:6-153, raft.py:112-123
 * No torch types appear here.  The Python host side (ptlflow_b200/_lib.py) binds these
 * symbols with ctypes; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - every function returns 0 on success, a negative pfb_status otherwise; the message is
 *     available from pfb_last_error() (thread local).  The Python shim raises RuntimeError,
 *     mirroring TORCH_CHECK in correlation.cpp:19-21.
 *   - nothing allocates: callers pass outputs and workspaces (sizes from pfb_*_bytes()).
 *   - everything is asynchronous on `stream` (the reference plugin launches on the legacy
 *     default stream, correlation_kernel.cu:278; here the caller's stream is explicit so
 *     CUDA-graph capture and torch's current stream both work).
 *   - activations are pixel-major ("NHWC"): [B, H, W, C] with C contiguous.  Coordinates and
 *     flow are always fp32 [B, H, W, 2] with (x, y) interleaved.
 *   - dtype is the STORAGE type of features / volume / activations / packed weights;
 *     accumulation, coordinates, bilinear weights, gates and softmax are always fp32.
 */
#ifndef PTLFLOW_B200_H_
#define PTLFLOW_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PFB_API __attribute__((visibility("default")))
#else
#define PFB_API
#endif

typedef void* pfb_stream; /* cudaStream_t */

typedef enum { PFB_F32 = 0, PFB_F16 = 1, PFB_BF16 = 2 } pfb_dtype;

typedef enum {
  PFB_OK = 0,
  PFB_ERR_ARG = -1,     /* bad argument (null pointer, unsupported size / dtype) */
  PFB_ERR_CUDA = -2,    /* a CUDA runtime / driver call failed */
  PFB_ERR_UNSUPPORTED = -3
} pfb_status;

#define PFB_MAX_LEVELS 8
#define PFB_MAX_SRC 4

PFB_API int pfb_version(void);
PFB_API const char* pfb_last_error(void);
/* sm major*10+minor of the current device, or negative status. */
PFB_API int pfb_device_arch(void);
/* A stream of the current device that belongs to the caller alone (cudaStreamNonBlocking).  The host side captures its CUDA
 * graphs on one: a stream handed out by a framework's stream pool can be the same underlying stream as one another host
 * thread is launching on, and that thread's work would land in the capture. */
PFB_API int pfb_stream_create(pfb_stream* out);
PFB_API int pfb_stream_destroy(pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a1 + a2: all-pairs correlation volume and its pooled pyramid
 *   replaces CorrBlock.corr + CorrBlock.__init__     ptlflow/models/raft/corr.py:13-27, 56-64
 * fmap1, fmap2 : [B, H, W, C] dtype.   pyramid[l] : [B*H*W, H>>l, W>>l] dtype (floor sizes),
 * level 0 = <f1, f2> / sqrt(C); level l = 2x2 mean of level l-1.
 * impl: 0 = auto (wgmma tensor-core GEMM for f16/bf16 when the shape allows, else SIMT),
 *       1 = force the SIMT fp32-accumulate kernel, 2 = force wgmma.
 * ---------------------------------------------------------------------------------- */
PFB_API int pfb_corr_volume_build(const void* fmap1, const void* fmap2, void* const* pyramid, int B, int H, int W,
                          int C, int levels, pfb_dtype dtype, int impl, pfb_stream stream);
/* Generalisation for the sibling corr.py copies (SURVEY.md appendix E): the queries are the H1 x W1 grid of fmap1, the targets
 * the H2 x W2 grid of fmap2 (SEA-RAFT builds one volume per level against a separately resized fmap2,
 * ptlflow/models/sea_raft/corr.py:77-83), and the scale is explicit (FlowFormer's cost volume is unscaled,
 * ptlflow/models/flowformer/encoder.py:543-561).  pyramid[l] : [B*H1*W1, H2>>l, W2>>l].
 * pfb_corr_volume_build(..., H, W, C, ...) == pfb_corr_volume_build_ex(..., H, W, H, W, C, levels, 1/sqrt(C), ...). */
PFB_API int pfb_corr_volume_build_ex(const void* fmap1, const void* fmap2, void* const* pyramid, int B, int H1, int W1, int H2, int W2,
                                     int C, int levels, float scale, pfb_dtype dtype, int impl, pfb_stream stream);
/* bytes of level l for the given feature-grid size (helper for callers that allocate). */
PFB_API size_t pfb_corr_level_bytes(int B, int H, int W, int level, pfb_dtype dtype);

/* ------------------------------------------------------------------------------------
 * a3: multi-scale radius-r lookup     replaces CorrBlock.__call__   corr.py:29-54
 * coords : [B, H, W, 2] fp32 absolute target coordinates (x, y).
 * out    : channel = l*(2r+1)^2 + i*(2r+1) + j, sample at (x/2^l + i - r, y/2^l + j - r)  (x-major).
 *          out_nchw = 0 -> [B, H, W, out_stride] (out_stride >= L*(2r+1)^2, extra channels zero-filled)
 *          out_nchw = 1 -> [B, L*(2r+1)^2, H, W]  (the corr-block protocol layout)
 * out_dtype may differ from the pyramid dtype (e.g. fp32 output from an fp16 volume).
 * ---------------------------------------------------------------------------------- */
PFB_API int pfb_corr_lookup(void* const* pyramid, const float* coords, void* out, int B, int H, int W, int levels,
                    int radius, pfb_dtype dtype, pfb_dtype out_dtype, int out_nchw, int out_stride,
                    pfb_stream stream);

/* Same with explicit level sizes (level_h[l] x level_w[l] instead of H>>l x W>>l): pyramids whose levels were built one by one
 * (pfb_corr_volume_build_ex) or whose target grid differs from the query grid.  level l is still sampled at coords / 2^l. */
PFB_API int pfb_corr_lookup_ex(void* const* pyramid, const int* level_h, const int* level_w, const float* coords, void* out, int B,
                               int H, int W, int levels, int radius, pfb_dtype dtype, pfb_dtype out_dtype, int out_nchw,
                               int out_stride, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a1 + a2 + a3 on the TILED pyramid (f16 / bf16 storage; what pfb_raft_refine uses with cfg.volume_layout = 1).
 * Level l of query q is ceil(h_l/4) x ceil(w_l/8) tiles of 4 rows x 8 columns (64 bytes = one DRAM access granule);
 * element (y, x) sits at element offset ((y>>2) * ceil(w_l/8) + (x>>3)) * 32 + (y&3) * 8 + (x&7) of the query's map.
 * A 10 x 10 lookup window touches 6.9 such tiles on average (442 B) where the dense layout costs 64 B of DRAM traffic
 * for every 20-byte window row (820 B).  Same values as pfb_corr_volume_build_ex / pfb_corr_lookup_ex, except that the
 * pooled levels are means of the fp32 products rounded once (the dense path rounds every level like the reference's
 * half model does).  pyramid[l]: pfb_corr_level_bytes_tiled(...) bytes, 16-byte aligned; out: [B,H1,W1,out_stride] dtype,
 * out_stride % 8 == 0, columns >= levels*(2r+1)^2 zero-filled.
 * ---------------------------------------------------------------------------------- */
PFB_API size_t pfb_corr_level_bytes_tiled(int B, int H1, int W1, int H2, int W2, int level);
PFB_API int pfb_corr_volume_build_tiled(const void* fmap1, const void* fmap2, void* const* pyramid, int B, int H1, int W1, int H2,
                                        int W2, int C, int levels, float scale, pfb_dtype dtype, pfb_stream stream);
PFB_API int pfb_corr_lookup_tiled(void* const* pyramid, const float* coords, void* out, int B, int H1, int W1, int H2, int W2,
                                  int levels, int radius, pfb_dtype dtype, int out_stride, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a4: on-the-fly correlation + lookup (no 4D volume)
 *   replaces AlternateCorrBlock.__call__     corr.py:78-101  (all levels, scaled by 1/sqrt(C))
 * fmap1 : [B, H, W, C];  fmap2_pyramid[l] : [B, H>>l, W>>l, C] (level 0 = fmap2, l>0 pooled by
 * pfb_avg_pool2x2_nhwc);  output as in pfb_corr_lookup.
 * ---------------------------------------------------------------------------------- */
PFB_API int pfb_corr_lookup_onthefly(const void* fmap1, void* const* fmap2_pyramid, const float* coords, void* out,
                             int B, int H, int W, int C, int levels, int radius, pfb_dtype dtype,
                             pfb_dtype out_dtype, int out_nchw, int out_stride, pfb_stream stream);
/* Same with an explicit scale of the dot products (0 = 1/sqrt(C)): features stored in rows wider than their real width (zero
 * channels up to a multiple of 64, MS-RAFT+'s 96-channel 1/4-scale features) keep the scale of the real width. */
PFB_API int pfb_corr_lookup_onthefly_ex(const void* fmap1, void* const* fmap2_pyramid, const float* coords, void* out, int B, int H, int W,
                                        int C, int levels, int radius, float scale, pfb_dtype dtype, pfb_dtype out_dtype, int out_nchw,
                                        int out_stride, pfb_stream stream);

/* a4 on the tensor cores (f16 / bf16, radius 4, C % 64 == 0, C <= 256, pixel-major output): every 8 x 16 tile of neighbouring queries
 * multiplies its query vectors with the region of fmap2_pyramid[l] that holds all its windows (wgmma GEMM, TMA-fed, out-of-map
 * targets zero-filled by the TMA unit) and blends its windows out of the accumulator; queries whose window does not fit the region
 * (rough flow inside a tile) are recomputed by the SIMT kernel of pfb_corr_lookup_onthefly, so the values never depend on the flow.
 * workspace: pfb_corr_lookup_onthefly_tc_workspace_bytes(B, H, W) bytes (one flag per query).  Same output as
 * pfb_corr_lookup_onthefly(..., out_nchw = 0) up to the storage-type rounding of the products. */
PFB_API size_t pfb_corr_lookup_onthefly_tc_workspace_bytes(int B, int H, int W);
PFB_API int pfb_corr_lookup_onthefly_tc(const void* fmap1, void* const* fmap2_pyramid, const float* coords, void* out, void* workspace,
                                        int B, int H, int W, int C, int levels, int radius, pfb_dtype dtype, int out_stride,
                                        pfb_stream stream);
/* Same with an explicit scale (0 = 1/sqrt(C)); the SIMT pass for the flagged queries uses the same scale. */
PFB_API int pfb_corr_lookup_onthefly_tc_ex(const void* fmap1, void* const* fmap2_pyramid, const float* coords, void* out, void* workspace,
                                           int B, int H, int W, int C, int levels, int radius, float scale, pfb_dtype dtype, int out_stride,
                                           pfb_stream stream);

/* The reference plugin's own entry point, same tensor contract:
 *   alt_cuda_corr.forward(fmap1, fmap2, coords, radius) -> [corr]     correlation.cpp:23-33
 * fmap1 [B,H1,W1,C], fmap2 [B,H2,W2,C], coords [B,1,H1,W1,2] fp32, out [B,1,(2r+1)^2,H1,W1];
 * unscaled dot products.  Unlike the reference (fp32 only, correlation_kernel.cu:278) the
 * features may be f16/bf16; out is `out_dtype`. */
PFB_API int pfb_alt_corr_forward(const void* fmap1, const void* fmap2, const float* coords, void* out, int B, int H1,
                         int W1, int H2, int W2, int C, int radius, pfb_dtype dtype, pfb_dtype out_dtype,
                         pfb_stream stream);

/* 2x2 mean pooling of a pixel-major tensor [N, H, W, C] -> [N, H/2, W/2, C] (floor). */
PFB_API int pfb_avg_pool2x2_nhwc(const void* in, void* out, int N, int H, int W, int C, pfb_dtype dtype,
                         pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * Convolution building block (stride 1, "same" zero padding, odd kernel), pixel-major.
 * The input is the channel-concatenation of up to PFB_MAX_SRC tensors, so torch.cat copies
 * of the reference (update.py:60,63,107,111,148) never happen.
 * ---------------------------------------------------------------------------------- */
typedef enum {
  PFB_EPI_LINEAR = 0,  /* out = scale * (acc + bias)                                        */
  PFB_EPI_RELU = 1,    /* out = relu(acc + bias)                                            */
  PFB_EPI_GRU_ZR = 2,  /* cols [0,hd): z = sigmoid -> aux_z;  cols [hd,2hd): r = sigmoid,
                          out = r * h                               update.py:61-63,68-70 */
  PFB_EPI_GRU_Q = 3,   /* q = tanh(acc+bias); out = (1 - z) * h + z * q     update.py:63-64 */
  PFB_EPI_FLOW = 4,    /* Cout = 2: coords1 += acc + bias (fp32, in place);
                          out(fp32) = coords1 - grid               raft.py:174-178          */
  PFB_EPI_RELU_APPEND_FLOW = 5, /* relu into cols [0,Cout) and copy flow(fp32 [.,2]) into the
                          next two columns                          update.py:111-112      */
  PFB_EPI_AXPY = 6,    /* out = residual + scale * (acc + bias); residual = aux_h[p * hidden + n]
                          (GMA Aggregate: fmap + gamma * attn@v)    gma_utils.py:101-113   */
  PFB_EPI_LINEAR_F32 = 7, /* out(fp32) = scale * (acc + bias): per-tap partial products of the flow head's
                          last convolution, summed over the 3x3 neighbourhood by pfb_flow_tap_gather */
  PFB_EPI_GELU = 8,    /* out = gelu(acc + bias), exact erf GELU (F.gelu default)   skflow/update.py:20-29 */
  PFB_EPI_RESIDUAL_GELU = 9, /* y = gelu(res + acc + bias), res = residual[p * residual_stride + residual_offset + n];
                          then, if post_w != NULL, out = gelu(y * (1 + post_w[n]) + post_b[n]) (a following depthwise
                          1x1 step x = gelu(x + dw1(x)) of a PCBlock, skflow/update.py:32-34), else out = y */
  PFB_EPI_LINEAR_APPEND_FLOW = 10 /* linear into cols [0,Cout) and flow (fp32 [.,2]) into the next two columns
                          (SKFlow motion encoder: cat[conv(cor_flo), flow], skflow/update.py:53-61) */
} pfb_epilogue;

typedef struct {
  const void* ptr; /* [B, H, W, stride] */
  int channels;    /* channels taken from this source */
  int stride;      /* elements per pixel in memory (>= offset + channels) */
  int offset;      /* first channel */
  int is_f32;      /* 1: fp32 source regardless of `dtype` (flow / coordinates) */
} pfb_conv_src;

typedef struct {
  pfb_conv_src src[PFB_MAX_SRC];
  int nsrc;
  int B, H, W;
  int KH, KW;          /* odd; padding KH/2, KW/2 */
  int Cout;            /* real output channels */
  int Cout_pad;        /* row length of the packed weight (>= Cout) */
  const void* weight;  /* packed by pfb_pack_conv_weight: [KH*KW][Cin_total][Cout_pad] dtype */
  const float* bias;   /* [Cout] fp32 (may be NULL) */
  int epilogue;        /* pfb_epilogue */
  float scale;         /* PFB_EPI_LINEAR only */
  void* out;           /* [B,H,W,out_stride] dtype (fp32 for PFB_EPI_FLOW) */
  int out_stride, out_offset;
  const void* aux_h;   /* GRU: hidden state [B,H,W,hd] dtype */
  void* aux_z;         /* GRU: z gate buffer [B,H,W,hd] dtype (written by ZR, read by Q) */
  int hidden;          /* hd */
  float* coords;       /* PFB_EPI_FLOW: coords1 [B,H,W,2] fp32 in/out */
  const float* flow;   /* PFB_EPI_RELU_APPEND_FLOW: [B,H,W,2] fp32 */
  pfb_dtype dtype;
  int impl;            /* 0 auto, 1 SIMT, 2 wgmma */
  /* tensor-core operand (f16/bf16 only, may be NULL -> SIMT path): the same weights packed K-major
   * by pfb_pack_conv_weight_kmajor: [KH*KW][Cout_pad_k][Cin_pad], every source padded to 64 channels */
  const void* weight_k;
  int Cin_pad, Cout_pad_k;
  /* optional per-pixel pre-activation term [B,H,W,addend_stride] dtype, added to the accumulator INSTEAD of `bias` before the
   * epilogue function (the iteration-invariant context part of the GRU gates: conv(inp) + bias, computed once per forward,
   * update.py:60-63 split by linearity).  addend_stride >= Cout_pad_k, % 8 == 0.  NULL = use bias. */
  const void* addend;
  int addend_stride;
  /* > 0 (1x1 layers, wgmma path): sample b multiplies with ITS OWN weight matrix, rows [b * w_rows_per_sample, + Cout_pad_k)
   * of weight_k [B * w_rows_per_sample][Cin_pad] -- one launch for all samples of "attention @ v" (gma_utils.py:101-113),
   * where the "weights" are the sample's transposed v.  0 = one weight matrix for all samples. */
  int w_rows_per_sample;
  /* PFB_EPI_RESIDUAL_GELU: the residual operand [B,H,W,residual_stride] dtype (fp32 when dtype is fp32), channels from
   * residual_offset, and the optional per-channel fp32 step post_w / post_b [Cout] (both NULL or both set) */
  const void* residual;
  int residual_stride, residual_offset;
  const float* post_w;
  const float* post_b;
} pfb_conv_params;

PFB_API int pfb_conv2d(const pfb_conv_params* p, pfb_stream stream);

/* torch-layout weight [Cout][Cin][KH][KW] (src_dtype) -> packed [KH*KW][Cin][Cout_pad] (dst_dtype),
 * written at column `col_offset` (so convz|convr share one packed matrix).  Columns outside
 * [col_offset, col_offset+Cout) are left untouched: zero the buffer first. */
PFB_API int pfb_pack_conv_weight(const void* src, void* dst, int Cout, int Cin, int KH, int KW, int Cout_pad,
                         int col_offset, pfb_dtype src_dtype, pfb_dtype dst_dtype, pfb_stream stream);
/* dst[offset + i] = (float) src[i] */
PFB_API int pfb_pack_bias(const void* src, float* dst, int n, int offset, pfb_dtype src_dtype, pfb_stream stream);
/* torch-layout weight -> K-major packing for the wgmma path: dst[tap][row_offset + co][kpos(ci)] where the
 * input channels are the concatenation of `nsrc` sources of src_channels[i] channels and each source is
 * padded to a multiple of 64 in dst (kpos skips the pad).  dst is [KH*KW][Cout_pad_k][Cin_pad]; zero it first. */
PFB_API int pfb_pack_conv_weight_kmajor(const void* src, void* dst, int Cout, int Cin, int KH, int KW, int Cout_pad_k,
                                        int row_offset, const int* src_channels, int nsrc, int Cin_pad,
                                        pfb_dtype src_dtype, pfb_dtype dst_dtype, pfb_stream stream);

/* Depthwise k x k convolution with its PCBlock residual and activation (skflow/update.py:32-33):
 *   out[p, c] = gelu(x[p, c] + bias[c] + sum_{ky, kx} weight[ky * k + kx][c] * x[p + (ky - k/2, kx - k/2), c])
 * stride 1, zero "same" padding, any odd k <= 31 (grids smaller than the kernel included), C % 2 == 0.
 * x: [B,H,W,in_stride] from channel in_offset; out: [B,H,W,out_stride] from out_offset (must not overlap x); offsets and
 * strides even.  weight [k*k][C], bias [C]: fp32.  dtype is the storage type of x / out; accumulation is fp32. */
PFB_API int pfb_depthwise_conv_gelu(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset,
                                    const float* weight, const float* bias, int B, int H, int W, int C, int k, pfb_dtype dtype,
                                    pfb_stream stream);

/* Depthwise k x k convolution followed by a LayerNorm over all C channels of each pixel, without the LayerNorm's affine part
 * (SEA-RAFT's ConvNextBlock, sea_raft/layer.py:71-75; the affine folds into the next 1x1 layer):
 *   y[p, c]   = bias[c] + sum_{ky, kx} weight[ky * k + kx][c] * x[p + (ky - k/2, kx - k/2), c]
 *   out[p, c] = (y[p, c] - mean_c y[p, .]) * rsqrt(var_c y[p, .] + eps)          (biased variance)
 * stride 1, zero "same" padding, any odd k <= 31, C even and <= 512.  Two passes: y is stored into `out` in the storage type, then
 * normalised in place with fp32 statistics (mean, then the variance about it).  x: [B,H,W,in_stride] from channel in_offset; out:
 * [B,H,W,out_stride] from out_offset (must not overlap x); offsets and strides even.  weight [k*k][C], bias [C]: fp32.  dtype is the
 * storage type of x / out; accumulation is fp32. */
PFB_API int pfb_depthwise_conv_layernorm(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset,
                                         const float* weight, const float* bias, int B, int H, int W, int C, int k, float eps,
                                         pfb_dtype dtype, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a10: upsampling
 *   convex 8x : RAFT.upsample_flow               ptlflow/models/raft/raft.py:112-123
 *   bilinear  : upflow8 (raft_small)             ptlflow/models/raft/utils.py:94-96
 * coords : [B,H,W,2] fp32 (flow = coords - grid);  mask : [B,H,W,576] dtype, channel =
 * tap*64 + sy*8 + sx, already scaled by 0.25.  out : [B, 2, out_h, out_w] fp32 (NCHW), the
 * window of the 8H x 8W result starting at (pad_top, pad_left) -- i.e. already un-padded.
 * flow_small (optional) : [B, 2, H, W] fp32.
 * ---------------------------------------------------------------------------------- */
PFB_API int pfb_convex_upsample(const float* coords, const void* mask, float* out, float* flow_small, int B, int H,
                        int W, int out_h, int out_w, int pad_top, int pad_left, pfb_dtype dtype,
                        pfb_stream stream);
PFB_API int pfb_upflow8(const float* coords, float* out, float* flow_small, int B, int H, int W, int out_h, int out_w,
                int pad_top, int pad_left, pfb_stream stream);

/* GMA attention: in-place softmax over the last axis of sim [rows, cols] (sim = pfb_corr_volume_build(q, k)
 * level 0: <q, k> / sqrt(dim_head) is exactly the content attention logit).   gma_utils.py:58-76 */
PFB_API int pfb_softmax_rows(void* x, size_t rows, int cols, pfb_dtype dtype, pfb_stream stream);
/* GMA attention with the relative-position term (position_only / position_and_content, gma_utils.py:6-30, 62-74).
 * Row r of attn [rows, H*W] (rows = heads * B * H*W, head-major) is the query i = r % (H*W) at grid row x = i / W, column y = i % W:
 *   attn[r][u*W + v] = softmax over (u, v) of  logits[r][u*W + v] + th[r*table_stride + u - x + P - 1] + tw[r*table_stride + v - y + P - 1]
 * logits [rows, H*W] dtype (content logits, may alias attn) or NULL (position only); th, tw fp32 per-query tables of 2P-1 entries
 * (scale * q . rel_height / rel_width), row stride table_stride >= 2P-1.  H, W <= P.  Softmax in fp32; each row is read once
 * and written once. */
PFB_API int pfb_attention_softmax_relpos(const void* logits, const float* th, const float* tw, size_t table_stride, void* attn,
                                         size_t rows, int H, int W, int P, pfb_dtype dtype, pfb_stream stream);
/* [B, HW, C] pixel-major -> [B, C, HW_pad] (zero padded): K-major operand for the attn @ v GEMM */
PFB_API int pfb_transpose_pm(const void* in, void* out, int B, int HW, int C, int HW_pad, pfb_dtype dtype, pfb_stream stream);

/* Flow head conv2 (3x3, C -> 2) as "1x1 GEMM to 18 tap-products, then gather": taps [B,H,W,tstride] fp32 holds
 * T[p][tap*2+o] = <W2[o,:,tap], x(p)>; delta(p)[o] = bias[o] + sum_tap T[p + tap][tap*2+o] (zero outside the image);
 * coords += delta, flow = coords - grid.        update.py:9,14 ; raft.py:174-178 */
PFB_API int pfb_flow_tap_gather(const float* taps, int tstride, const float* bias, float* coords, float* flow, int B, int H, int W,
                                pfb_stream stream);

/* cnet output [B,H,W,hd+cd] -> net = tanh(first hd), inp = relu(rest)     raft.py:155-158 */
PFB_API int pfb_context_split(const void* cnet, void* net, void* inp, int B, int H, int W, int hidden, int context,
                      pfb_dtype dtype, pfb_stream stream);
/* coords[b,y,x] = (x, y) + (flow_init ? flow_init[b,:,y,x] (NCHW fp32) : 0)   raft.py:103-110,162-167 */
PFB_API int pfb_init_coords(float* coords, const float* flow_init_nchw, int B, int H, int W, pfb_stream stream);
/* Warm start (SURVEY.md section 8(f) rank 4): forward_interpolate of ptlflow/utils/external/raft.py:155-185 /
 * ptlflow/utils/utils.py:454-478 (scipy griddata(method="nearest") on the CPU there) on the device.
 * flow_nchw, out_nchw: fp32 [B,2,H,W]; exact nearest neighbour in fp64, ties to the lowest source index. */
PFB_API int pfb_forward_interpolate(const float* flow_nchw, float* out_nchw, int B, int H, int W, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a6-a9, a11: the refinement loop   (BasicUpdateBlock / SmallUpdateBlock + RAFT.forward loop)
 *   ptlflow/models/raft/update.py:115-153, ptlflow/models/raft/raft.py:170-192
 * ---------------------------------------------------------------------------------- */
typedef enum {
  PFB_L_CONVC1 = 0, PFB_L_CONVC2, PFB_L_CONVF1, PFB_L_CONVF2, PFB_L_CONV,
  PFB_L_GRU_ZR1, PFB_L_GRU_Q1, PFB_L_GRU_ZR2, PFB_L_GRU_Q2,
  PFB_L_FLOW1, PFB_L_FLOW2, PFB_L_MASK1, PFB_L_MASK2,
  PFB_L_AGG_V, /* GMA Aggregate.to_v (1x1, no bias) */
  PFB_L_FLOW2T, /* flow_head.conv2 re-expressed as a 1x1 layer with 18 = 9 taps x 2 outputs (row = tap*2+o) */
  /* round 2 (tensor-core path only; present iff weight_k != NULL, else the loop uses the layers above):
   * the context (`inp`) columns of the four GRU convolutions as their own layers, evaluated ONCE per forward ... */
  PFB_L_CTX_ZR1, PFB_L_CTX_Q1, PFB_L_CTX_ZR2, PFB_L_CTX_Q2,
  /* ... the same four without those columns (sources: hidden state | motion features), evaluated every iteration ... */
  PFB_L_GRUX_ZR1, PFB_L_GRUX_Q1, PFB_L_GRUX_ZR2, PFB_L_GRUX_Q2,
  /* ... and convc2 (256 -> 192) | convf2 (128 -> 64) as ONE block-diagonal 3x3 layer 384 -> 256 (update.py:98-102): N = 256
   * runs the tensor core at its nominal rate, the two separate layers (N = 192, 64) do not */
  PFB_L_CONVC2F2,
  PFB_L_AGG_PROJ, /* GMA Aggregate.project (1x1, heads*128 -> 128, no bias); present iff num_heads > 1 */
  PFB_L_COUNT
} pfb_layer_id;

typedef struct {
  const void* weight; /* packed, see pfb_pack_conv_weight */
  const float* bias;
  int Cout, Cout_pad, Cin, KH, KW;
  const void* weight_k; /* K-major packing (wgmma), NULL if not packed */
  int Cin_pad, Cout_pad_k;
} pfb_layer;

typedef struct {
  int variant;        /* 0 = raft (BasicUpdateBlock, SepConvGRU, convex upsample)
                         1 = raft_small (SmallUpdateBlock, ConvGRU, bilinear upflow8)
                         2 = gma (GMAUpdateBlock: raft + per-iteration attention aggregate, gma/update.py:127-160)
                         (3 skflow, 4 sea_raft, 5 ms_raft_plus, 6 ccmr: their own entry points only) */
  pfb_dtype dtype;
  int B, H, W;        /* 1/8-resolution grid */
  int feat_dim;       /* C of fmap1/fmap2 (on-the-fly mode) */
  int corr_levels, corr_radius;
  int hidden_dim, context_dim;
  int iters;
  int alternate_corr; /* 0: look up the materialised pyramid; 1: on-the-fly (a4) */
  int out_h, out_w, pad_top, pad_left; /* full-resolution output window */
  int impl;           /* 0 auto, 1 SIMT everywhere, 2 wgmma where available */
  int volume_layout;  /* 0: dense pyramid (pfb_corr_volume_build); 1: tiled pyramid (pfb_corr_volume_build_tiled) */
  int fork_flow;      /* 1: the flow branch of the motion encoder (convf1, convf2) and the once-per-forward context terms run on a second
                         stream of the calling host thread, forked / joined with events (parallel branches when the caller captures a
                         CUDA graph); 0: everything on `stream`.  Half-precision tensor path only, ignored elsewhere. */
  int num_heads;      /* gma: attention heads (0 is read as 1); > 1 needs layer PFB_L_AGG_PROJ */
} pfb_raft_cfg;

typedef struct {
  pfb_layer layers[PFB_L_COUNT];
} pfb_raft_weights;

typedef struct {
  void* const* pyramid;       /* [corr_levels] volume levels, or (alternate_corr) fmap2 levels */
  const void* fmap1;          /* alternate_corr only */
  void* net;                  /* [B,H,W,hidden] dtype, in/out */
  const void* inp;            /* [B,H,W,context] dtype */
  float* coords;              /* [B,H,W,2] fp32, in/out (absolute target coordinates) */
  float* flow_up;             /* [B,2,out_h,out_w] fp32 */
  float* flow_small;          /* [B,2,H,W] fp32 */
  void* workspace;            /* pfb_raft_workspace_bytes(cfg) */
  size_t workspace_bytes;
  const void* attention;      /* gma: softmax attention [heads, B, H*W, H*W] dtype, head-major (pfb_softmax_rows or
                                 pfb_attention_softmax_relpos) */
  float agg_gamma;            /* gma: Aggregate.gamma */
} pfb_raft_buffers;

PFB_API size_t pfb_raft_workspace_bytes(const pfb_raft_cfg* cfg);
/* Runs cfg->iters refinement iterations followed by the final upsample.  Only the last
 * iteration evaluates the mask head (raft.py:192 returns only the last prediction in eval). */
PFB_API int pfb_raft_refine(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                    pfb_stream stream);
/* One update iteration without the upsample (used by the operator-level parity tests);
 * mask_out may be NULL. Lookup output ("corr") is taken from `corr` if non-NULL, otherwise
 * computed from buf->pyramid. */
PFB_API int pfb_raft_update_iter(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf,
                         const void* corr, void* mask_out, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a15: SKFlow's refinement loop (SKUpdateBlock6_Deep_nopoolres_AllDecoder + the GMA loop)
 *   ptlflow/models/skflow/update.py:7-99, ptlflow/models/skflow/skflow.py:197-232
 * pfb_raft_cfg with variant = 3 (accepted by the pfb_skflow_* entry points only), hidden = context = 128, any num_heads;
 * pfb_raft_buffers as for gma (attention and agg_gamma are required).
 * ---------------------------------------------------------------------------------- */
#define PFB_SK_MAX_DW 8
/* PCBlock4_Deep_nopool_res(C_in, C_out, k_conv), every activation padded to C = align(C_in, 32) channels whose padding stays
 * exactly zero (zero weights and biases), the FFN hidden width to hid = align(int(1.5 * C_in), 32):
 *   x = gelu(x + ffn1b(gelu(ffn1a(x))));  x = gelu(x + dw_k(x)) for k in k_conv;  x = gelu(x + pw(x));  out = ffn2b(gelu(ffn2a(x)))
 * ffn1a: 1x1 C -> hid, ffn1b: hid -> C, pw: C -> C, ffn2a: C -> hid, ffn2b: hid -> C_out (pfb_layer packing as in the raft
 * loop).  dw_weight[i] [k*k][C], dw_bias[i] [C] fp32.  When dw_k[0] == 1 that step rides ffn1b's epilogue. */
typedef struct {
  pfb_layer ffn1a, ffn1b, pw, ffn2a, ffn2b;
  int C, hid;
  int n_dw;
  int dw_k[PFB_SK_MAX_DW];
  const float* dw_weight[PFB_SK_MAX_DW];
  const float* dw_bias[PFB_SK_MAX_DW];
} pfb_pc_block;

typedef enum {
  PFB_SK_CONVC1 = 0, /* encoder.convc1: planes -> 256 (followed by a GELU) */
  PFB_SK_CONVC2,     /* encoder.convc2: 256 -> 192 */
  PFB_SK_CONVF2,     /* encoder.convf2: 128 -> 64 */
  PFB_SK_CONV,       /* encoder.conv: 256 -> 126 (+ flow) */
  PFB_SK_GRU,        /* gru: [net | inp | motion | motion_global] 512 -> 128, k_conv = PCUpdater_conv */
  PFB_SK_FLOW_HEAD,  /* flow_head: 128 -> 2 */
  PFB_SK_BLOCKS
} pfb_skflow_block_id;

typedef struct {
  pfb_pc_block blocks[PFB_SK_BLOCKS];
  pfb_layer convf1;           /* encoder.convf1: 1x1 2 -> 128 on the fp32 flow, no activation */
  pfb_layer mask1, mask2;     /* mask.0 (3x3 128 -> 256, ReLU), mask.2 (1x1 256 -> 576, x0.25) */
  pfb_layer agg_v, agg_proj;  /* aggregator.to_v, aggregator.project (num_heads > 1) */
} pfb_skflow_weights;

PFB_API size_t pfb_skflow_workspace_bytes(const pfb_raft_cfg* cfg);
/* cfg->iters update iterations, then the convex upsample (mask head on the last iteration only). */
PFB_API int pfb_skflow_refine(const pfb_raft_cfg* cfg, const pfb_skflow_weights* w, const pfb_raft_buffers* buf, pfb_stream stream);
/* One update iteration without the upsample; corr (pixel-major [B,H,W,corr_stride], columns past the planes zero, where
 * corr_stride = align(planes, 32)) replaces the lookup when non-NULL; mask_out [B,H,W,576] may be NULL. */
PFB_API int pfb_skflow_update_iter(const pfb_raft_cfg* cfg, const pfb_skflow_weights* w, const pfb_raft_buffers* buf,
                                   const void* corr, void* mask_out, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a16: SEA-RAFT's refinement loop (BasicUpdateBlock of ConvNeXt blocks + the SEARAFT.forward loop)
 *   ptlflow/models/sea_raft/update.py:18-54, layer.py:41-83, sea_raft.py:189-236
 * pfb_raft_cfg with variant = 4 (accepted by the pfb_searaft_* entry points only), hidden = context = 128.  The correlation pyramid
 * is RAFT's (SEA-RAFT's per-level volumes against a bilinearly halved fmap2 are exactly the 2x2-pooled levels), so `pyramid`,
 * `fmap1` and alternate_corr mean what they mean for pfb_raft_refine.
 * ---------------------------------------------------------------------------------- */
#define PFB_SR_MAX_BLOCKS 8
/* One ConvNextBlock(384 -> 128) on x = [net | context | motion | flow]:
 *   x^ = LayerNorm(dw_k(x)) without affine (pfb_depthwise_conv_layernorm);  h = gelu(pw1(x^));  net' = out([h | x])
 * pw1: 1x1 384 -> 512 = pwconv1 with the LayerNorm affine folded in (W1 diag(ln_w), b1 + W1 ln_b);
 * out: 1x1 [h (512) | x (384)] -> 128 = final(x + gamma * pwconv2(h)) as one layer ([Wf diag(gamma) W2 | Wf], Wf (gamma b2) + bf). */
typedef struct {
  int dw_k;
  const float* dw_weight; /* [k*k][384] fp32 */
  const float* dw_bias;   /* [384] fp32 */
  pfb_layer pw1, out;
} pfb_convnext_block;

typedef struct {
  pfb_layer init_conv;                      /* 3x3 256 -> 256, no activation (sea_raft.py:105) */
  pfb_layer convc1, convc2, convf1, convf2, conv;  /* motion encoder, as RAFT's (update.py:18-36) */
  int num_blocks;
  pfb_convnext_block blocks[PFB_SR_MAX_BLOCKS];
  float ln_eps;                             /* LayerNorm eps (1e-6) */
  pfb_layer flow1;                          /* flow_head.0: 3x3 128 -> 256, ReLU */
  pfb_layer flow2;                          /* flow_head.2 restricted to its flow outputs: 3x3 256 -> 2 */
  pfb_layer flow2t;                         /* the same as a 1x1 layer to the 9 x 2 tap products (PFB_L_FLOW2T), or weight = NULL */
  pfb_layer mask1, mask2;                   /* upsample_weight.0 (3x3 128 -> 256, ReLU), upsample_weight.2 (1x1 256 -> 576, x0.25) */
} pfb_searaft_weights;

PFB_API size_t pfb_searaft_workspace_bytes(const pfb_raft_cfg* cfg);
/* The whole SEA-RAFT forward after the encoders: init_conv on buf->inp (the context network's output [B,H,W,256]), the initial
 * flow head at coords = buf->coords (the grid on entry), cfg->iters update iterations (none when iters = 0: no pyramid is read),
 * the mask head on the final net and the convex upsample.  buf->net [B,H,W,128] receives the final net; buf->coords the final
 * coordinates. */
PFB_API int pfb_searaft_refine(const pfb_raft_cfg* cfg, const pfb_searaft_weights* w, const pfb_raft_buffers* buf, pfb_stream stream);
/* One update iteration without the upsample: buf->net [B,H,W,128] in/out, buf->inp the context [B,H,W,128], buf->coords in/out;
 * corr (pixel-major [B,H,W,planes]) replaces the lookup when non-NULL; mask_out [B,H,W,576] may be NULL. */
PFB_API int pfb_searaft_update_iter(const pfb_raft_cfg* cfg, const pfb_searaft_weights* w, const pfb_raft_buffers* buf,
                                    const void* corr, void* mask_out, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a17: MS-RAFT+'s four-scale refinement (ptlflow/models/ms_raft_plus/ms_raft_plus.py:146-226)
 * The scale loop runs RAFT's update block (pfb_raft_weights with CONVC1.Cin = levels*(2r+1)^2 and MASK2.Cout = 36) once per scale
 * (1/16, 1/8, 1/4, 1/2), with pfb_raft_cfg variant = 5 (accepted by the pfb_msraft_* entry points only) describing that scale's
 * grid.  pyramid / fmap1 / alternate_corr / volume_layout mean what they mean for pfb_raft_refine.
 * ---------------------------------------------------------------------------------- */
/* out [B,2H,2W,Cs+Ck] = cat[bilinear 2x (align_corners = False, edge clamped) of src [B,H,W,Cs], skip [B,2H,2W,Ck]] along the
 * channels: TF.resize + torch.cat of the encoders' up path (extractor.py:193-210).  Cs, Ck multiples of 8 (Ck may be 0, skip
 * NULL); 16-byte aligned pointers. */
PFB_API int pfb_upsample2x_concat(const void* src, int src_channels, const void* skip, int skip_channels, void* out, int B, int H, int W,
                                  pfb_dtype dtype, pfb_stream stream);
/* Convex 2x upsample (upsample_flow with scale = 2, ms_raft_plus.py:138-149): mask [B,H,W,36] dtype, channel = tap*4 + sy*2 + sx,
 * already scaled by 0.25; softmax over the 9 taps; the 3x3 neighbourhood of 2 * value is unfolded with ZERO padding.
 *   mode 0: value = coords - grid; out [B,2,out_h,out_w] fp32, the window of the 2H x 2W result at (pad_top, pad_left)
 *   mode 1: value = coords (absolute, the handover between scales); out [B,2H,2W,2] fp32 pixel-major; window arguments unused */
PFB_API int pfb_convex_upsample2x(const float* coords, const void* mask, float* out, int mode, int B, int H, int W, int out_h, int out_w,
                                  int pad_top, int pad_left, pfb_dtype dtype, pfb_stream stream);
/* downflow (ms_raft_plus.py:22-35): flow [B,2,H,W] fp32 -> out [B,2,out_h,out_w], bilinear with align_corners = True, u scaled by
 * out_w / W and v by out_h / H. */
PFB_API int pfb_downflow(const float* flow, float* out, int B, int H, int W, int out_h, int out_w, pfb_stream stream);
PFB_API size_t pfb_msraft_workspace_bytes(const pfb_raft_cfg* cfg);
/* One scale: cfg->iters >= 1 update iterations from buf->coords (absolute, this scale's grid), the GRU context terms once, the mask
 * head on the last iteration only.  corr_scale: the on-the-fly lookup's scale, 0 = 1/sqrt(feat_dim).  Then either
 *   next_coords != NULL: pfb_convex_upsample2x mode 1 into next_coords [B,2H,2W,2] (the next scale's starting coordinates), or
 *   next_coords == NULL: mode 0 into buf->flow_up (cfg out_h / out_w / pad window) and, if buf->flow_small != NULL, pfb_downflow
 *                        of it into buf->flow_small [B,2,out_h/16,out_w/16]. */
PFB_API int pfb_msraft_refine(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf, float corr_scale,
                              float* next_coords, pfb_stream stream);
/* One update iteration without the upsample; corr (pixel-major [B,H,W,planes]) replaces the lookup when non-NULL; mask_out
 * [B,H,W,36] may be NULL. */
PFB_API int pfb_msraft_update_iter(const pfb_raft_cfg* cfg, const pfb_raft_weights* w, const pfb_raft_buffers* buf, const void* corr,
                                   void* mask_out, float corr_scale, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * a18: CCMR / CCMR+ (ptlflow/models/ccmr/ccmr.py:141-230): MS-RAFT+'s scale loop with XCiT global context (xcit.py:58-427).
 * ---------------------------------------------------------------------------------- */
/* The handover between scales (ccmr.py:195-202): pfb_convex_upsample2x of value = coords - grid, with zero-padded taps, plus the fine
 * grid: out [B,2H,2W,2] fp32 pixel-major = the next scale's starting coordinates. */
PFB_API int pfb_convex_handover2x(const float* coords, const void* mask, float* out, int B, int H, int W, pfb_dtype dtype, pfb_stream stream);
/* Row LayerNorm over C channels (C even, <= 512) of P pixels, biased variance, fp32 statistics; x [P,in_stride] from in_offset, out
 * [P,out_stride] from out_offset (may alias x exactly); gamma / beta fp32 [C] (both NULL: no affine). */
PFB_API int pfb_layernorm(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset, const float* gamma,
                          const float* beta, size_t P, int C, float eps, pfb_dtype dtype, pfb_stream stream);
/* Depthwise 3x3 convolution, zero "same" padding, y = dw(x) + bias (weight fp32 [9][C] tap-major, bias fp32 [C]), then
 *   mode 0: out = gelu(y);   mode 1: out = y + addend[p, addend_offset + c]  (addend [B,H,W,addend_stride], storage type)
 * The two convolutions of LPI (xcit.py:98-139).  Strides / offsets even, C even; out must not overlap x. */
PFB_API int pfb_depthwise_conv3x3_ex(const void* x, int in_stride, int in_offset, void* out, int out_stride, int out_offset,
                                     const float* weight, const float* bias, const void* addend, int addend_stride, int addend_offset,
                                     int B, int H, int W, int C, int mode, pfb_dtype dtype, pfb_stream stream);
/* PositionalEncodingFourier's features (xcit.py:58-95) before token_projection, computed in fp32 and rounded once:
 * out [H,W,64] storage type, channels 0..31 from the row index, 32..63 from the column index. */
PFB_API int pfb_fourier_features(void* out, int H, int W, pfb_dtype dtype, pfb_stream stream);
/* XCA statistics (xcit.py:167-186) of q = qk[., q_offset + h*16 + i], k = qk[., k_offset + h*16 + j] over the N = H*W pixels of each
 * sample: per (sample, head) the 16 x 16 gram sum_n q_i k_j and the column sums of squares of q and k.  qk [B,N,qk_stride] storage
 * type.  stats [B][2304] fp32: gram at h*256 + i*16 + j, sum q^2 at 2048 + c, sum k^2 at 2176 + c.  Each CTA sums 512 pixels in fp32,
 * the partials are combined in a fixed order in fp64: the result does not depend on scheduling.
 * workspace: pfb_xca_stats_workspace_bytes(B, N). */
PFB_API size_t pfb_xca_stats_workspace_bytes(int B, int N);
PFB_API int pfb_xca_stats(const void* qk, int qk_stride, int q_offset, int k_offset, int B, int N, float* stats, void* workspace,
                          pfb_dtype dtype, pfb_stream stream);
/* Folds the 8-head XCA into one linear layer per sample: A_h = softmax_j(temperature[h] * gram_ij / (max(|q_i|, 1e-12) max(|k_j|,
 * 1e-12))) in fp32, then  W_b = proj_w blockdiag(A_1..A_8) v_w,  bias_b = proj_w blockdiag(A) v_b + proj_b  (v_w, proj_w fp32
 * [128][128] row-major [out][in], v_b, proj_b fp32 [128]).  w_out [B][128 in][128 out] (the pfb_pack_conv_weight layout of a 1x1
 * layer), w_out_k [B*128 out][128 in] (K-major, may be NULL): storage type; bias_out [B][128] fp32. */
PFB_API int pfb_xca_fold(const float* stats, const float* temperature, const float* v_w, const float* v_b, const float* proj_w,
                         const float* proj_b, void* w_out, void* w_out_k, float* bias_out, int B, pfb_dtype dtype, pfb_stream stream);
/* upflow2 (ccmr/utils.py:97-99): 2 * bilinear 2x (align_corners = True) of flow [B,2,H,W] fp32 into out [B,2,out_h,out_w] fp32, the
 * window of the 2H x 2W result at (pad_top, pad_left). */
PFB_API int pfb_upflow2(const float* flow, float* out, int B, int H, int W, int out_h, int out_w, int pad_top, int pad_left,
                        pfb_stream stream);

/* One XCABlock of embed_dim 128, 8 heads, mlp_ratio 1 (xcit.py:242-300), folded for inference.  The LayerNorms' eps is ln_eps. */
typedef struct {
  pfb_layer pos_proj;          /* pos_embeder.token_projection: 1x1 64 -> 128 with bias */
  pfb_layer qk;                /* q | k (1x1 128 -> 256) on norm1's output, norm1's affine folded in */
  const float* v_weight;       /* [128][128] fp32: W_v diag(norm1.weight) */
  const float* v_bias;         /* [128]: W_v norm1.bias + b_v */
  const float* proj_weight;    /* [128][128]: diag(gamma1) W_proj */
  const float* proj_bias;      /* [128]: gamma1 * b_proj */
  const float* temperature;    /* [8] */
  const float* ln3_weight;     /* norm3 affine [128] (applied: LPI's convolutions are zero padded) */
  const float* ln3_bias;
  const float* dw1_weight;     /* local_mp.conv1 [9][128] tap-major, bias [128] */
  const float* dw1_bias;
  const float* gn_weight;      /* local_mp.bn: GroupNorm(8, 128) */
  const float* gn_bias;
  const float* dw2_weight;     /* local_mp.conv2 times gamma3 [9][128], bias times gamma3 [128] */
  const float* dw2_bias;
  pfb_layer fc1;               /* mlp.fc1 (128 -> 128, GELU) with norm2's affine folded in */
  pfb_layer fc2;               /* diag(gamma2) mlp.fc2 */
  float ln_eps, gn_eps;
} pfb_xcit_block;

typedef struct {
  pfb_raft_weights raft;        /* the update block: MS-RAFT+'s layers with the GRU over [h | inp | motion | motion_global] */
  pfb_xcit_block context;       /* xcit[i]: self-attention on inp -> global_context */
  pfb_xcit_block aggregator;    /* update_block.aggregator[i]: q, k from global_context, v from the motion features */
} pfb_ccmr_weights;

/* The whole XCiT (xcit.py:406-427) of one scale's context: x = inp + pos; x = block(x) -> out [B,H,W,128].  cfg describes the scale
 * (variant 6); workspace: pfb_ccmr_workspace_bytes(cfg). */
PFB_API int pfb_xcit_context(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const void* inp, void* out, void* workspace,
                             size_t workspace_bytes, pfb_stream stream);
PFB_API size_t pfb_ccmr_workspace_bytes(const pfb_raft_cfg* cfg);
/* One scale (pfb_raft_cfg variant 6, accepted by the pfb_ccmr_* entry points only): the global context of buf->inp and the aggregator's
 * folded attention once, the GRU context terms once, cfg->iters >= 1 iterations (lookup, motion encoder, aggregator written into the
 * motion_global columns of the GRU input, GRU, flow head), the mask head on the last one.  Then either
 *   next_coords != NULL: pfb_convex_handover2x into next_coords [B,2H,2W,2], or
 *   next_coords == NULL: the convex 2x of the flow, followed by `upflow2` (0 or 1) pfb_upflow2 steps, into buf->flow_up (cfg's window
 *                        of the result) and, if buf->flow_small != NULL, pfb_downflow of it into [B,2,out_h/16,out_w/16]. */
PFB_API int pfb_ccmr_refine(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf, float corr_scale, int upflow2,
                            float* next_coords, pfb_stream stream);
/* One update iteration after the scale's global context (no upsample); corr (pixel-major [B,H,W,planes]) replaces the lookup when
 * non-NULL; mask_out [B,H,W,36] may be NULL. */
PFB_API int pfb_ccmr_update_iter(const pfb_raft_cfg* cfg, const pfb_ccmr_weights* w, const pfb_raft_buffers* buf, const void* corr,
                                 void* mask_out, float corr_scale, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * Encoder-side kernels (SURVEY.md section 8(f) rank 1: the callers either side of the path).
 * The first 7x7 convolution and the residual blocks' stride-1 3x3 convolutions of BasicEncoder (extractor.py:122-267)
 * run here, the strided, 1x1 and bottleneck convolutions in cuDNN; pre-processing, instance norm + ReLU (+ residual)
 * and the residual joins are fused here.
 * ---------------------------------------------------------------------------------- */
/* images [B,2,3,H,W] BGR in [0,1] (NCHW) -> out [2B,Hp,Wp,out_channels] pixel-major RGB in [-1,1], replicate
 * padded; channels 3..out_channels-1 are zero (out_channels = 4 gives the first convolution 8-byte pixels, which
 * saves cuDNN its own channel-padding pass).  The first B entries are frame 1, the next B frame 2.
 * raft.py:127-135, base_model.py:206-246 */
PFB_API int pfb_preprocess_frames(const void* images, void* out, int B, int H, int W, int Hp, int Wp, int pad_top,
                                  int pad_left, int out_channels, pfb_dtype dtype, pfb_stream stream);
/* y = act(IN(x)) or, with residual, y = relu(residual + act(IN(x)));  x, y, residual: [B,H,W,C].
 * IN = nn.InstanceNorm2d defaults (no affine, biased variance, eps).   extractor.py:29-31,52-58 */
PFB_API size_t pfb_instance_norm_workspace_bytes(int B, int C);
PFB_API int pfb_instance_norm_act(const void* x, void* y, const void* residual, void* workspace, int B, int H, int W, int C,
                                  float eps, int relu, pfb_dtype dtype, pfb_stream stream);
/* Same, for sums already accumulated into the workspace by the producing kernel (pfb_first_conv7x7s2):
 * workspace = B*C*2 doubles (sum, sum of squares; zeroed by the caller before the producer ran) + B*C float2. */
PFB_API int pfb_instance_norm_apply(const void* x, void* y, const void* residual, void* workspace, int B, int H, int W, int C,
                                    float eps, int relu, pfb_dtype dtype, pfb_stream stream);
/* Group norm (nn.GroupNorm) of x + bias: statistics per (image, group of group_size consecutive channels), biased variance, then
 * gamma / beta per channel; y = act(GN(x + bias)) or, with residual, relu(residual + act(GN(x + bias))).  bias (the producing
 * convolution's, fp32 [C]), gamma, beta (fp32 [C]) may each be NULL.  group_size = 1 without bias and affine is instance norm.
 * workspace: pfb_instance_norm_workspace_bytes(B, C).  C % 8 == 0, C <= 512, group_size divides C. */
PFB_API int pfb_group_norm_act(const void* x, void* y, const void* residual, void* workspace, const float* bias, const float* gamma,
                               const float* beta, int B, int H, int W, int C, int group_size, float eps, int relu, pfb_dtype dtype,
                               pfb_stream stream);
/* The same from per-(image, channel) sums of x already in the workspace (pfb_first_conv7x7s2's stats output). */
PFB_API int pfb_group_norm_apply(const void* x, void* y, const void* residual, void* workspace, const float* bias, const float* gamma,
                                 const float* beta, int B, int H, int W, int C, int group_size, float eps, int relu, pfb_dtype dtype,
                                 pfb_stream stream);
/* First encoder convolution: nn.Conv2d(3, 64, 7, stride=2, padding=3) of BasicEncoder (extractor.py:136,171-178)
 * on wgmma without an im2col buffer (overlapping-window operand descriptors, see csrc/first_conv.cu).
 *   x      [N,H,W,4]  f16/bf16 pixel-major frames from pfb_preprocess_frames(out_channels = 4); H, W even
 *   wpack  9 x 8192 B: for input-row offset j = 0..8 a [128][32] K-major tile, row p*64+co, column 4*t+c =
 *          W[co][c][j-2p][t-1] (zero where j-2p or t-1 fall outside 0..6, or c = 3), stored as non-swizzled wgmma
 *          core matrices [16 row groups][4 K groups][8 rows][8 elements]   (ptlflow_b200.ops.pack_first_conv)
 *   bias   fp32 [64] or NULL (folded batch norm + conv bias);  relu: apply max(.,0) after the bias
 *   stats  NULL, or B*64*2 doubles that receive per (image, channel) sum / sum of squares of the fp32 result
 *          (instance norm: follow with pfb_instance_norm_apply)
 *   out    [N,H/2,W/2,64] */
/* convf1 of the motion encoder, nn.Conv2d(2, 128, 7, padding=3) + ReLU on the fp32 flow (update.py:84,96), on
 * wgmma with the same overlapping-window operand (csrc/first_conv.cu).  The flow is split into hi + lo halves of
 * the storage type inside the kernel, so the arithmetic equals fp32 flow x f16/bf16 weights, fp32 accumulate.
 *   flow   fp32 [B,H,W,2];   bias fp32 [128]
 *   wpack  7 x 16384 B: for filter row ky a [128][64] K-major tile, column 8*t+c = W[co][c & 1][ky][t-1] for
 *          c < 4 (hi and lo halves see the same weight), zero for t = 0 or c >= 4; non-swizzled wgmma core-matrix
 *          order [16 row groups][8 K groups][8 rows][8 elements]   (ptlflow_b200.ops.pack_flow_conv)
 *   out    [B,H,W,out_stride] storage type, channels out_offset .. out_offset+127 written */
PFB_API int pfb_flow_conv7x7(const float* flow, const void* wpack, const float* bias, void* out, int out_stride, int out_offset,
                             int B, int H, int W, pfb_dtype dtype, pfb_stream stream);
PFB_API int pfb_first_conv7x7s2(const void* x, const void* wpack, const float* bias, void* out, double* stats, int N, int H, int W,
                                int relu, pfb_dtype dtype, pfb_stream stream);
/* 3x3 stride-1 "same" convolution of the encoders' residual blocks on wgmma, output channels on the MMA's M dimension
 * (csrc/enc_conv_umma.cu).
 *   x         [B,H,W,Cin] f16/bf16 pixel-major, contiguous; Cin a multiple of 32
 *   weight_k  the K-major packing of ptlflow_b200.ops.PackedConv: [9][Cout_pad_k][Cin_pad], Cout_pad_k = Cout rounded up to
 *             32, Cin_pad = Cin rounded up to 64 (zero columns beyond Cin)
 *   Cout      64, 96 or 128
 *   epilogue  PFB_ENC_CONV_LINEAR: acc (bias ignored; instance norm follows);  PFB_ENC_CONV_BIAS_RELU: relu(acc + bias);
 *             PFB_ENC_CONV_BIAS_RELU_RESIDUAL: relu(residual + relu(acc + bias)), residual [B,H,W,Cout] contiguous
 *   bias      fp32 [Cout]
 *   out       [B,H,W,out_stride], channels out_offset .. out_offset + Cout - 1 written (both multiples of 8)
 * Accumulation in fp32, one rounding to the storage type. */
enum pfb_enc_conv_epilogue { PFB_ENC_CONV_LINEAR = 0, PFB_ENC_CONV_BIAS_RELU = 1, PFB_ENC_CONV_BIAS_RELU_RESIDUAL = 2 };
/* 1 when pfb_enc_conv3x3 runs these channel counts in this storage type (host only, no device needed). */
PFB_API int pfb_enc_conv3x3_supported(int Cin, int Cout, pfb_dtype dtype);
PFB_API int pfb_enc_conv3x3(const void* x, const void* weight_k, const float* bias, const void* residual, void* out, int B, int H,
                            int W, int Cin, int Cout, int out_stride, int out_offset, int epilogue, pfb_dtype dtype,
                            pfb_stream stream);
/* y = act(x + bias[c]) or, with residual, y = relu(residual + act(x + bias[c]));  bias fp32 [C] (may be NULL);
 * workspace >= 8*C bytes.  Used for the batch-norm-folded context encoder (conv bias + BN shift) and conv2. */
PFB_API int pfb_bias_act(const void* x, const float* bias, const void* residual, void* y, void* workspace, int B, int H, int W,
                         int C, int relu, pfb_dtype dtype, pfb_stream stream);

/* ------------------------------------------------------------------------------------
 * Measurement hooks (bench.py): launch accounting and live per-kernel-class timing.
 * kernel_class: 0 volume, 1 pool, 2 lookup, 3 on-the-fly lookup, 4 update-block conv (wgmma / SIMT), 5 upsample,
 * 6 misc (packing, coords, softmax, transposes), 7 encoder normalise / bias / activation passes, 8 encoder instance-norm
 * statistics, 9 first encoder convolution (wgmma), 10 convf1 (7x7 on the flow, wgmma), 11 flow-head tap gather,
 * 12 depthwise convolution (SKFlow), 13 depthwise convolution + LayerNorm (SEA-RAFT); -1 = all.  pfb_profile_collect synchronises
 * the device, writes summed milliseconds and span counts per class (arrays of >= PFB_KERNEL_CLASSES entries) and clears the
 * recorded spans.
 * ---------------------------------------------------------------------------------- */
#define PFB_KERNEL_CLASSES 14
PFB_API unsigned long long pfb_launch_count(int kernel_class);
PFB_API int pfb_profile_enable(int on);
PFB_API int pfb_profile_collect(double* ms, unsigned long long* n, int len);

#ifdef __cplusplus
}
#endif
#endif /* PTLFLOW_B200_H_ */
