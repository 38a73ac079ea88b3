"""Tensor-level wrappers over the C ABI (plumbing only: pointers, shapes, current stream).

Layout conventions (see include/ptlflow_b200.h): feature / activation tensors are pixel-major
``[B, H, W, C]``; coordinates are fp32 ``[B, H, W, 2]`` with (x, y) interleaved.  Helpers at the
bottom convert from/to the reference's NCHW tensors without a copy when the tensor is already
channels_last.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import threading
from typing import List, NamedTuple, Optional, Sequence

import torch

from . import _lib
from ._lib import check, dtype_code, load, ptr_array, require_cuda, stream_ptr


# ------------------------------------------------------------------------------------------
# layout helpers
# ------------------------------------------------------------------------------------------
def to_pixel_major(x: torch.Tensor) -> torch.Tensor:
    """NCHW (any memory format) -> contiguous [B,H,W,C]; free when x is channels_last."""
    return x.permute(0, 2, 3, 1).contiguous()


def coords_to_pixel_major(coords: torch.Tensor) -> torch.Tensor:
    """[B,2,H,W] any float dtype -> fp32 [B,H,W,2]."""
    return coords.permute(0, 2, 3, 1).float().contiguous()


# ------------------------------------------------------------------------------------------
# a1 + a2
# ------------------------------------------------------------------------------------------
def alloc_pyramid(B: int, H: int, W: int, levels: int, dtype: torch.dtype, device) -> List[torch.Tensor]:
    return [torch.empty((B * H * W, H >> l, W >> l), dtype=dtype, device=device) for l in range(levels)]


def corr_volume_build(fmap1: torch.Tensor, fmap2: torch.Tensor, levels: int = 4, impl: int = 0,
                      out: Optional[Sequence[torch.Tensor]] = None) -> List[torch.Tensor]:
    """fmap [B,H,W,C] -> [level0 [B*H*W,H,W], ..., level L-1].  ptlflow/models/raft/corr.py:13-27,56-64."""
    require_cuda(fmap1, "fmap1"); require_cuda(fmap2, "fmap2")
    if fmap1.shape != fmap2.shape or fmap1.dtype != fmap2.dtype or fmap1.dim() != 4:
        raise RuntimeError("corr_volume_build: fmap1/fmap2 must be [B,H,W,C] with equal shape and dtype")
    B, H, W, Cc = fmap1.shape
    if (H >> (levels - 1)) < 1 or (W >> (levels - 1)) < 1:
        raise RuntimeError(f"corr_volume_build: {H}x{W} grid too small for {levels} levels")
    pyr = list(out) if out is not None else alloc_pyramid(B, H, W, levels, fmap1.dtype, fmap1.device)
    with torch.cuda.device(fmap1.device):
        check(load().pfb_corr_volume_build(fmap1.data_ptr(), fmap2.data_ptr(), ptr_array(pyr), B, H, W, Cc, levels,
                                           dtype_code(fmap1.dtype), impl, stream_ptr(fmap1.device)), "corr_volume_build")
    return pyr


def corr_volume_build_ex(fmap1: torch.Tensor, fmap2: torch.Tensor, levels: int = 1, scale: Optional[float] = None,
                         impl: int = 0) -> List[torch.Tensor]:
    """fmap1 [B,H1,W1,C] (queries), fmap2 [B,H2,W2,C] (targets, any grid) -> [level0 [B*H1*W1,H2,W2], ...]; ``scale`` defaults to
    1/sqrt(C).  SEA-RAFT's per-level volumes (sea_raft/corr.py:77-83), FlowFormer's unscaled cost maps (encoder.py:543-561)."""
    require_cuda(fmap1, "fmap1"); require_cuda(fmap2, "fmap2")
    if fmap1.dim() != 4 or fmap2.dim() != 4 or fmap1.shape[0] != fmap2.shape[0] or fmap1.shape[3] != fmap2.shape[3] or fmap1.dtype != fmap2.dtype:
        raise RuntimeError("corr_volume_build_ex: fmap1 [B,H1,W1,C] / fmap2 [B,H2,W2,C] with equal B, C and dtype")
    B, H1, W1, Cc = fmap1.shape
    _, H2, W2, _ = fmap2.shape
    if (H2 >> (levels - 1)) < 1 or (W2 >> (levels - 1)) < 1:
        raise RuntimeError(f"corr_volume_build_ex: {H2}x{W2} target grid too small for {levels} levels")
    pyr = [torch.empty((B * H1 * W1, H2 >> l, W2 >> l), dtype=fmap1.dtype, device=fmap1.device) for l in range(levels)]
    with torch.cuda.device(fmap1.device):
        check(load().pfb_corr_volume_build_ex(fmap1.data_ptr(), fmap2.data_ptr(), ptr_array(pyr), B, H1, W1, H2, W2, Cc, levels,
                                              float(Cc ** -0.5 if scale is None else scale), dtype_code(fmap1.dtype), impl,
                                              stream_ptr(fmap1.device)), "corr_volume_build_ex")
    return pyr


# ------------------------------------------------------------------------------------------
# a1 + a2 + a3 on the tiled pyramid (see include/ptlflow_b200.h: 4 x 8 tiles of 64 bytes)
# ------------------------------------------------------------------------------------------
def tiled_supported(fmap: torch.Tensor, levels: int) -> bool:
    return fmap.dtype in (torch.float16, torch.bfloat16) and fmap.shape[-1] % 64 == 0 and fmap.shape[-1] <= 256 and 1 <= levels <= 4


def corr_volume_build_tiled(fmap1: torch.Tensor, fmap2: torch.Tensor, levels: int = 4, scale: Optional[float] = None) -> List[torch.Tensor]:
    """fmap1 [B,H1,W1,C], fmap2 [B,H2,W2,C] (f16/bf16) -> per level a flat tensor [B*H1*W1, tiles_y*tiles_x*32] in the tiled layout."""
    require_cuda(fmap1, "fmap1"); require_cuda(fmap2, "fmap2")
    B, H1, W1, Cc = fmap1.shape
    _, H2, W2, _ = fmap2.shape
    if fmap1.dtype != fmap2.dtype or fmap2.shape[0] != B or fmap2.shape[3] != Cc:
        raise RuntimeError("corr_volume_build_tiled: fmap1 / fmap2 must agree in batch, channels and dtype")
    lib = load()
    pyr = []
    for l in range(levels):
        nbytes = lib.pfb_corr_level_bytes_tiled(B, H1, W1, H2, W2, l)
        if nbytes == 0:
            raise RuntimeError(f"corr_volume_build_tiled: {H2}x{W2} target grid too small for {levels} levels")
        pyr.append(torch.empty((B * H1 * W1, nbytes // (2 * B * H1 * W1)), dtype=fmap1.dtype, device=fmap1.device))
    with torch.cuda.device(fmap1.device):
        check(lib.pfb_corr_volume_build_tiled(fmap1.data_ptr(), fmap2.data_ptr(), ptr_array(pyr), B, H1, W1, H2, W2, Cc, levels,
                                              float(Cc ** -0.5 if scale is None else scale), dtype_code(fmap1.dtype),
                                              stream_ptr(fmap1.device)), "corr_volume_build_tiled")
    return pyr


def untile_level(level: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """Tiled level [Q, tiles_y*tiles_x*32] -> dense [Q, h, w] (pure indexing; tests and debugging)."""
    ty, tx = (h + 3) // 4, (w + 7) // 8
    v = level.view(level.shape[0], ty, tx, 4, 8).permute(0, 1, 3, 2, 4).reshape(level.shape[0], ty * 4, tx * 8)
    return v[:, :h, :w].contiguous()


def corr_lookup_tiled(pyramid: Sequence[torch.Tensor], coords: torch.Tensor, radius: int, targets_hw, out_stride: Optional[int] = None) -> torch.Tensor:
    """coords fp32 [B,H1,W1,2] -> [B,H1,W1,out_stride] in the pyramid's dtype (pixel-major, the refinement loop's layout)."""
    require_cuda(coords, "coords")
    if coords.dtype != torch.float32:
        raise RuntimeError("corr_lookup_tiled: coords must be float32 [B,H,W,2]")
    B, H, W, _ = coords.shape
    L = len(pyramid)
    planes = L * (2 * radius + 1) ** 2
    stride = (planes + 7) // 8 * 8 if out_stride is None else out_stride
    out = torch.empty((B, H, W, stride), dtype=pyramid[0].dtype, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_corr_lookup_tiled(ptr_array(pyramid), coords.data_ptr(), out.data_ptr(), B, H, W, targets_hw[0], targets_hw[1], L,
                                           radius, dtype_code(pyramid[0].dtype), stride, stream_ptr(coords.device)), "corr_lookup_tiled")
    return out


# ------------------------------------------------------------------------------------------
# a3
# ------------------------------------------------------------------------------------------
def corr_lookup(pyramid: Sequence[torch.Tensor], coords: torch.Tensor, radius: int, grid_hw, nchw: bool = True,
                out_dtype: Optional[torch.dtype] = None, out_stride: Optional[int] = None, level_hw=None) -> torch.Tensor:
    """coords fp32 [B,H,W,2] -> [B, L*(2r+1)^2, H, W] (nchw) or [B,H,W,out_stride].  corr.py:29-54.
    ``level_hw``: explicit (h, w) per level when the levels are not the floor-halved query grid."""
    require_cuda(coords, "coords")
    if coords.dtype != torch.float32:
        raise RuntimeError("corr_lookup: coords must be float32 [B,H,W,2]")
    B, H, W, _ = coords.shape
    assert (H, W) == tuple(grid_hw)
    L = len(pyramid)
    planes = L * (2 * radius + 1) ** 2
    odt = out_dtype or pyramid[0].dtype
    stride = planes if out_stride is None else out_stride
    out = torch.empty((B, planes, H, W) if nchw else (B, H, W, stride), dtype=odt, device=coords.device)
    with torch.cuda.device(coords.device):
        if level_hw is None:
            check(load().pfb_corr_lookup(ptr_array(pyramid), coords.data_ptr(), out.data_ptr(), B, H, W, L, radius,
                                         dtype_code(pyramid[0].dtype), dtype_code(odt), int(nchw), stride,
                                         stream_ptr(coords.device)), "corr_lookup")
        else:
            lh = (C.c_int * L)(*[int(h) for h, _ in level_hw])
            lw = (C.c_int * L)(*[int(w) for _, w in level_hw])
            check(load().pfb_corr_lookup_ex(ptr_array(pyramid), lh, lw, coords.data_ptr(), out.data_ptr(), B, H, W, L, radius,
                                            dtype_code(pyramid[0].dtype), dtype_code(odt), int(nchw), stride,
                                            stream_ptr(coords.device)), "corr_lookup_ex")
    return out


# ------------------------------------------------------------------------------------------
# a4
# ------------------------------------------------------------------------------------------
def avg_pool2x2(x: torch.Tensor) -> torch.Tensor:
    """[N,H,W,C] -> [N,H/2,W/2,C]."""
    require_cuda(x, "x")
    N, H, W, Cc = x.shape
    out = torch.empty((N, H // 2, W // 2, Cc), dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        check(load().pfb_avg_pool2x2_nhwc(x.data_ptr(), out.data_ptr(), N, H, W, Cc, dtype_code(x.dtype), stream_ptr(x.device)), "avg_pool2x2")
    return out


def feature_pyramid(fmap2: torch.Tensor, levels: int) -> List[torch.Tensor]:
    """fmap2 [B,H,W,C] and its pooled copies (AlternateCorrBlock.__init__, corr.py:67-76)."""
    pyr = [fmap2]
    for _ in range(levels - 1):
        pyr.append(avg_pool2x2(pyr[-1]))
    return pyr


def corr_lookup_onthefly(fmap1: torch.Tensor, fmap2_pyramid: Sequence[torch.Tensor], coords: torch.Tensor,
                         radius: int, nchw: bool = True, out_dtype: Optional[torch.dtype] = None,
                         out_stride: Optional[int] = None) -> torch.Tensor:
    require_cuda(fmap1, "fmap1"); require_cuda(coords, "coords")
    B, H, W, Cc = fmap1.shape
    L = len(fmap2_pyramid)
    planes = L * (2 * radius + 1) ** 2
    odt = out_dtype or fmap1.dtype
    stride = planes if out_stride is None else out_stride
    out = torch.empty((B, planes, H, W) if nchw else (B, H, W, stride), dtype=odt, device=fmap1.device)
    with torch.cuda.device(fmap1.device):
        check(load().pfb_corr_lookup_onthefly(fmap1.data_ptr(), ptr_array(fmap2_pyramid), coords.data_ptr(), out.data_ptr(),
                                              B, H, W, Cc, L, radius, dtype_code(fmap1.dtype), dtype_code(odt), int(nchw),
                                              stride, stream_ptr(fmap1.device)), "corr_lookup_onthefly")
    return out


def corr_lookup_onthefly_tc(fmap1: torch.Tensor, fmap2_pyramid: Sequence[torch.Tensor], coords: torch.Tensor, radius: int = 4,
                            out_stride: Optional[int] = None) -> torch.Tensor:
    """a4 on the tensor cores: fmap1 [B,H,W,C] f16/bf16, fmap2 levels, coords fp32 [B,H,W,2] -> pixel-major [B,H,W,out_stride]."""
    require_cuda(fmap1, "fmap1"); require_cuda(coords, "coords")
    B, H, W, Cc = fmap1.shape
    L = len(fmap2_pyramid)
    planes = L * (2 * radius + 1) ** 2
    stride = (planes + 7) // 8 * 8 if out_stride is None else out_stride
    out = torch.empty((B, H, W, stride), dtype=fmap1.dtype, device=fmap1.device)
    lib = load()
    ws = torch.empty(max(1, lib.pfb_corr_lookup_onthefly_tc_workspace_bytes(B, H, W)), dtype=torch.uint8, device=fmap1.device)
    with torch.cuda.device(fmap1.device):
        check(lib.pfb_corr_lookup_onthefly_tc(fmap1.data_ptr(), ptr_array(fmap2_pyramid), coords.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                              B, H, W, Cc, L, radius, dtype_code(fmap1.dtype), stride, stream_ptr(fmap1.device)),
              "corr_lookup_onthefly_tc")
    out._pfb_flags = ws  # (tests read how many queries took the SIMT pass)
    return out


# ------------------------------------------------------------------------------------------
# conv building block
# ------------------------------------------------------------------------------------------
class ConvWeights(NamedTuple):
    """A weight / bias pair shaped like an nn.Conv2d's, for PackedConv: slices, folds and repacks of a model's parameters."""

    weight: torch.Tensor
    bias: Optional[torch.Tensor] = None


class PackedConv:
    """One (possibly fused) conv layer: packed weight [KH*KW][Cin][Cout_pad] + fp32 bias."""

    def __init__(self, convs, dtype: torch.dtype, device, cout_align: int = 8, src_channels=None):
        """``src_channels`` (list of the concatenated sources' channel counts) additionally builds the K-major
        packing [KH*KW][Cout_pad_k][Cin_pad] consumed by the wgmma kernels (f16 / bf16 only)."""
        convs = list(convs)
        w0 = convs[0].weight
        self.Cin, self.KH, self.KW = w0.shape[1], w0.shape[2], w0.shape[3]
        for c in convs:
            assert tuple(c.weight.shape[1:]) == (self.Cin, self.KH, self.KW)
        self.Cout = sum(c.weight.shape[0] for c in convs)
        self.Cout_pad = (self.Cout + cout_align - 1) // cout_align * cout_align
        self.dtype = dtype
        self.weight = torch.zeros((self.KH * self.KW, self.Cin, self.Cout_pad), dtype=dtype, device=device)
        self.weight_k, self.Cin_pad, self.Cout_pad_k = None, 0, 0
        if src_channels is not None and dtype != torch.float32:
            assert sum(src_channels) == self.Cin
            self.Cin_pad = sum((c + 63) // 64 * 64 for c in src_channels)
            self.Cout_pad_k = (self.Cout + 31) // 32 * 32 if self.Cout > 16 else 16
            self.weight_k = torch.zeros((self.KH * self.KW, self.Cout_pad_k, self.Cin_pad), dtype=dtype, device=device)
        self.bias = torch.zeros((max(self.Cout_pad, self.Cout_pad_k, 32),), dtype=torch.float32, device=device)
        lib = load()
        off = 0
        with torch.cuda.device(device):
            for c in convs:
                w = c.weight.detach().to(device).contiguous()
                check(lib.pfb_pack_conv_weight(w.data_ptr(), self.weight.data_ptr(), w.shape[0], self.Cin, self.KH, self.KW,
                                               self.Cout_pad, off, dtype_code(w.dtype), dtype_code(dtype), stream_ptr(device)), "pack_conv_weight")
                if self.weight_k is not None:
                    sc = (C.c_int * len(src_channels))(*src_channels)
                    check(lib.pfb_pack_conv_weight_kmajor(w.data_ptr(), self.weight_k.data_ptr(), w.shape[0], self.Cin, self.KH, self.KW,
                                                          self.Cout_pad_k, off, sc, len(src_channels), self.Cin_pad,
                                                          dtype_code(w.dtype), dtype_code(dtype), stream_ptr(device)), "pack_conv_weight_kmajor")
                if c.bias is not None:
                    bsrc = c.bias.detach().to(device).contiguous()
                    check(lib.pfb_pack_bias(bsrc.data_ptr(), self.bias.data_ptr(), bsrc.numel(), off, dtype_code(bsrc.dtype), stream_ptr(device)), "pack_bias")
                off += w.shape[0]

    def layer_struct(self) -> _lib.Layer:
        return _lib.Layer(self.weight.data_ptr(), self.bias.data_ptr(), self.Cout, self.Cout_pad, self.Cin, self.KH, self.KW,
                          self.weight_k.data_ptr() if self.weight_k is not None else None, self.Cin_pad, self.Cout_pad_k)


def conv2d(srcs, packed: PackedConv, out: torch.Tensor, epilogue: int = _lib.EPI_LINEAR, out_offset: int = 0,
           scale: float = 1.0, aux_h=None, aux_z=None, hidden: int = 0, coords=None, flow=None, impl: int = 0,
           residual=None, post_w: Optional[torch.Tensor] = None, post_b: Optional[torch.Tensor] = None,
           addend: Optional[torch.Tensor] = None, w_rows_per_sample: int = 0) -> torch.Tensor:
    """srcs: list of tensors [B,H,W,Ci] or (tensor, channels, offset) triples.  Mostly for tests.
    ``residual`` (EPI_RESIDUAL_GELU): a tensor [B,H,W,Cr] or a (tensor, offset) pair; ``post_w`` / ``post_b``: fp32 [Cout].
    ``addend``: a per-pixel term [B,H,W,S] (S >= Cout_pad_k) added instead of the bias.  ``w_rows_per_sample`` > 0 (1x1 layers):
    sample b multiplies with rows [b * w_rows_per_sample, + Cout_pad_k) of ``packed.weight_k`` viewed as [B * w_rows_per_sample,
    Cin_pad].  Both are served by the wgmma path only."""
    p = _lib.ConvParams()
    first = srcs[0][0] if isinstance(srcs[0], tuple) else srcs[0]
    B, H, W = first.shape[:3]
    for i, s in enumerate(srcs):
        t, ch, off = s if isinstance(s, tuple) else (s, s.shape[-1], 0)
        require_cuda(t, f"src{i}")
        p.src[i] = _lib.ConvSrc(t.data_ptr(), ch, t.shape[-1], off, int(t.dtype == torch.float32 and packed.dtype != torch.float32))
    p.nsrc = len(srcs)
    p.B, p.H, p.W, p.KH, p.KW = B, H, W, packed.KH, packed.KW
    p.Cout, p.Cout_pad = packed.Cout, packed.Cout_pad
    p.weight, p.bias = packed.weight.data_ptr(), packed.bias.data_ptr()
    p.epilogue, p.scale = epilogue, scale
    p.out, p.out_stride, p.out_offset = out.data_ptr(), out.shape[-1], out_offset
    p.aux_h = aux_h.data_ptr() if aux_h is not None else None
    p.aux_z = aux_z.data_ptr() if aux_z is not None else None
    p.hidden = hidden
    p.coords = coords.data_ptr() if coords is not None else None
    p.flow = flow.data_ptr() if flow is not None else None
    p.dtype, p.impl = dtype_code(packed.dtype), impl
    p.weight_k = packed.weight_k.data_ptr() if packed.weight_k is not None else None
    p.Cin_pad, p.Cout_pad_k = packed.Cin_pad, packed.Cout_pad_k
    if residual is not None:
        rt, roff = residual if isinstance(residual, tuple) else (residual, 0)
        require_cuda(rt, "residual")
        p.residual, p.residual_stride, p.residual_offset = rt.data_ptr(), rt.shape[-1], roff
    if post_w is not None:
        p.post_w, p.post_b = post_w.data_ptr(), post_b.data_ptr()
    if addend is not None:
        require_cuda(addend, "addend")
        p.addend, p.addend_stride = addend.data_ptr(), addend.shape[-1]
    p.w_rows_per_sample = w_rows_per_sample
    with torch.cuda.device(out.device):
        check(load().pfb_conv2d(C.byref(p), stream_ptr(out.device)), "conv2d")
    return out


def enc_conv3x3_supported(cin: int, cout: int, dtype: torch.dtype) -> bool:
    """Whether enc_conv3x3 runs a 3x3 stride-1 convolution with these channel counts in this storage type (host only)."""
    if dtype not in (torch.float16, torch.bfloat16):
        return False
    return bool(load().pfb_enc_conv3x3_supported(int(cin), int(cout), dtype_code(dtype)))


def enc_conv3x3(x: torch.Tensor, packed: PackedConv, epilogue: int = _lib.ENC_CONV_LINEAR, bias: Optional[torch.Tensor] = None,
                residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, out_offset: int = 0) -> torch.Tensor:
    """3x3 stride-1 "same" convolution x [B,H,W,Cin] -> [B,H,W,Cout] on pfb_enc_conv3x3 (see the header).  ``packed``: a
    PackedConv with the K-major packing (src_channels given); ``bias`` fp32 [Cout] (the epilogues with bias); ``residual``
    [B,H,W,Cout] (ENC_CONV_BIAS_RELU_RESIDUAL).  ``out`` [B,H,W,S] receives channels out_offset .. out_offset + Cout - 1."""
    require_cuda(x, "x")
    B, H, W, Cin = x.shape
    if packed.weight_k is None or (packed.KH, packed.KW) != (3, 3) or packed.Cin != Cin or not x.is_contiguous() or x.dtype != packed.dtype:
        raise RuntimeError("enc_conv3x3: x must be contiguous [B,H,W,Cin] in the dtype of a 3x3 PackedConv with the K-major packing")
    if out is None:
        out = torch.empty((B, H, W, packed.Cout), dtype=x.dtype, device=x.device)
    require_cuda(out, "out")
    if out.shape[:3] != x.shape[:3] or not out.is_contiguous() or out.dtype != x.dtype:
        raise RuntimeError("enc_conv3x3: out must be contiguous [B,H,W,S] in the input's dtype")
    if bias is not None and (bias.dtype != torch.float32 or bias.numel() < packed.Cout or not bias.is_cuda):
        raise RuntimeError("enc_conv3x3: bias must be fp32 [Cout] on the device")
    if residual is not None and (tuple(residual.shape) != (B, H, W, packed.Cout) or not residual.is_contiguous() or residual.dtype != x.dtype):
        raise RuntimeError("enc_conv3x3: residual must be contiguous [B,H,W,Cout] in the input's dtype")
    with torch.cuda.device(x.device):
        check(load().pfb_enc_conv3x3(x.data_ptr(), packed.weight_k.data_ptr(), bias.data_ptr() if bias is not None else None,
                                     residual.data_ptr() if residual is not None else None, out.data_ptr(), B, H, W, Cin, packed.Cout,
                                     out.shape[-1], out_offset, epilogue, dtype_code(x.dtype), stream_ptr(x.device)), "enc_conv3x3")
    return out


def depthwise_conv_gelu(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, k: int, channels: Optional[int] = None,
                        in_offset: int = 0, out: Optional[torch.Tensor] = None, out_offset: int = 0) -> torch.Tensor:
    """gelu(x + depthwise_conv_kxk(x) + bias) of a PCBlock (skflow/update.py:32-33).  x [B,H,W,Cs] pixel-major, the ``channels``
    channels from ``in_offset``; weight fp32 [k*k, C] (tap-major), bias fp32 [C].  Returns [B,H,W,C] (or writes ``out`` from
    ``out_offset``)."""
    require_cuda(x, "x")
    B, H, W, Cs = x.shape
    Cc = Cs - in_offset if channels is None else channels
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=x.dtype, device=x.device)
    require_cuda(out, "out")
    if weight.dtype != torch.float32 or bias.dtype != torch.float32 or tuple(weight.shape) != (k * k, Cc) or bias.numel() != Cc:
        raise RuntimeError("depthwise_conv_gelu: weight must be fp32 [k*k, C] and bias fp32 [C]")
    with torch.cuda.device(x.device):
        check(load().pfb_depthwise_conv_gelu(x.data_ptr(), Cs, in_offset, out.data_ptr(), out.shape[-1], out_offset, weight.data_ptr(),
                                             bias.data_ptr(), B, H, W, Cc, k, dtype_code(x.dtype), stream_ptr(x.device)),
              "depthwise_conv_gelu")
    return out


def depthwise_conv_layernorm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, k: int, channels: Optional[int] = None,
                             in_offset: int = 0, eps: float = 1e-6, out: Optional[torch.Tensor] = None, out_offset: int = 0) -> torch.Tensor:
    """LayerNorm over the channels (no affine) of depthwise_conv_kxk(x) + bias: SEA-RAFT's ConvNextBlock before pwconv1
    (sea_raft/layer.py:71-75).  x [B,H,W,Cs] pixel-major, the ``channels`` channels from ``in_offset``; weight fp32 [k*k, C]
    (tap-major), bias fp32 [C].  Returns [B,H,W,C] (or writes ``out`` from ``out_offset``)."""
    require_cuda(x, "x")
    B, H, W, Cs = x.shape
    Cc = Cs - in_offset if channels is None else channels
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=x.dtype, device=x.device)
    require_cuda(out, "out")
    if weight.dtype != torch.float32 or bias.dtype != torch.float32 or tuple(weight.shape) != (k * k, Cc) or bias.numel() != Cc:
        raise RuntimeError("depthwise_conv_layernorm: weight must be fp32 [k*k, C] and bias fp32 [C]")
    require_cuda(weight, "weight"); require_cuda(bias, "bias")
    with torch.cuda.device(x.device):
        check(load().pfb_depthwise_conv_layernorm(x.data_ptr(), Cs, in_offset, out.data_ptr(), out.shape[-1], out_offset, weight.data_ptr(),
                                                  bias.data_ptr(), B, H, W, Cc, k, eps, dtype_code(x.dtype), stream_ptr(x.device)),
              "depthwise_conv_layernorm")
    return out


# ------------------------------------------------------------------------------------------
# a10 and small helpers
# ------------------------------------------------------------------------------------------
def convex_upsample(coords: torch.Tensor, mask: torch.Tensor, out_hw=None, pad=(0, 0)):
    """coords fp32 [B,H,W,2], mask [B,H,W,576] -> (flow_up fp32 [B,2,oh,ow], flow_small fp32 [B,2,H,W])."""
    require_cuda(coords, "coords"); require_cuda(mask, "mask")
    B, H, W, _ = coords.shape
    oh, ow = out_hw or (8 * H, 8 * W)
    up = torch.empty((B, 2, oh, ow), dtype=torch.float32, device=coords.device)
    small = torch.empty((B, 2, H, W), dtype=torch.float32, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_convex_upsample(coords.data_ptr(), mask.data_ptr(), up.data_ptr(), small.data_ptr(), B, H, W, oh, ow,
                                         pad[0], pad[1], dtype_code(mask.dtype), stream_ptr(coords.device)), "convex_upsample")
    return up, small


def upflow8(coords: torch.Tensor, out_hw=None, pad=(0, 0)):
    require_cuda(coords, "coords")
    B, H, W, _ = coords.shape
    oh, ow = out_hw or (8 * H, 8 * W)
    up = torch.empty((B, 2, oh, ow), dtype=torch.float32, device=coords.device)
    small = torch.empty((B, 2, H, W), dtype=torch.float32, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_upflow8(coords.data_ptr(), up.data_ptr(), small.data_ptr(), B, H, W, oh, ow, pad[0], pad[1],
                                 stream_ptr(coords.device)), "upflow8")
    return up, small


def softmax_rows(x: torch.Tensor) -> torch.Tensor:
    """In-place softmax over the last axis of a 2-D tensor (GMA attention, gma_utils.py:74)."""
    require_cuda(x, "x")
    rows, cols = x.shape
    with torch.cuda.device(x.device):
        check(load().pfb_softmax_rows(x.data_ptr(), rows, cols, dtype_code(x.dtype), stream_ptr(x.device)), "softmax_rows")
    return x


def attention_softmax_relpos(logits: Optional[torch.Tensor], th: torch.Tensor, tw: torch.Tensor, H: int, W: int, P: int,
                             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GMA attention with the relative-position term (gma_utils.py:6-30, 62-74): row r of the result ([rows, H*W], rows =
    heads*B*H*W head-major) is softmax over (u, v) of ``logits[r, u*W+v] + th[r, u-x+P-1] + tw[r, v-y+P-1]`` for the query
    (x, y) = divmod(r % (H*W), W).  ``logits``: content logits in the storage dtype or None (position only); may be ``out``.
    ``th``, ``tw``: fp32 [rows, 2P-1] views with unit column stride and one shared row stride."""
    if not (th.is_cuda and tw.is_cuda):
        raise RuntimeError("attention_softmax_relpos: th / tw must be CUDA tensors")
    rows = th.shape[0]
    if th.dtype != torch.float32 or tw.dtype != torch.float32 or th.shape != (rows, 2 * P - 1) or tw.shape != th.shape \
            or th.stride() != tw.stride() or th.stride(1) != 1:
        raise RuntimeError("attention_softmax_relpos: th / tw must be fp32 [rows, 2P-1] views with equal strides")
    if logits is not None:
        require_cuda(logits, "logits")
        if logits.shape != (rows, H * W):
            raise RuntimeError(f"attention_softmax_relpos: logits {tuple(logits.shape)} != ({rows}, {H * W})")
    if out is None:
        out = torch.empty((rows, H * W), dtype=logits.dtype if logits is not None else torch.float32, device=th.device)
    require_cuda(out, "out")
    if logits is not None and out.dtype != logits.dtype:
        raise RuntimeError("attention_softmax_relpos: logits and out must share the storage dtype")
    with torch.cuda.device(th.device):
        check(load().pfb_attention_softmax_relpos(logits.data_ptr() if logits is not None else None, th.data_ptr(), tw.data_ptr(),
                                                  th.stride(0), out.data_ptr(), rows, H, W, P, dtype_code(out.dtype),
                                                  stream_ptr(th.device)), "attention_softmax_relpos")
    return out


def init_coords(B: int, H: int, W: int, device, flow_init: Optional[torch.Tensor] = None) -> torch.Tensor:
    coords = torch.empty((B, H, W, 2), dtype=torch.float32, device=device)
    fi = None
    if flow_init is not None:
        fi = flow_init.to(device=device, dtype=torch.float32).contiguous()
    with torch.cuda.device(device):
        check(load().pfb_init_coords(coords.data_ptr(), fi.data_ptr() if fi is not None else None, B, H, W, stream_ptr(device)), "init_coords")
    return coords


def forward_interpolate(flow: torch.Tensor) -> torch.Tensor:
    """flow [B,2,H,W] on CUDA -> forward-warped, nearest-filled flow [B,2,H,W] fp32 (warm start)."""
    require_cuda(flow, "flow")
    f = flow.detach().to(torch.float32).contiguous()
    B, two, H, W = f.shape
    if two != 2:
        raise RuntimeError("forward_interpolate: expected [B,2,H,W]")
    out = torch.empty_like(f)
    with torch.cuda.device(f.device):
        check(load().pfb_forward_interpolate(f.data_ptr(), out.data_ptr(), B, H, W, stream_ptr(f.device)), "forward_interpolate")
    return out


def context_split(cnet: torch.Tensor, hidden: int, context: int):
    """cnet [B,H,W,hidden+context] -> (tanh(net), relu(inp)) pixel-major.  raft.py:155-158."""
    require_cuda(cnet, "cnet")
    B, H, W, Cc = cnet.shape
    assert Cc == hidden + context
    net = torch.empty((B, H, W, hidden), dtype=cnet.dtype, device=cnet.device)
    inp = torch.empty((B, H, W, context), dtype=cnet.dtype, device=cnet.device)
    with torch.cuda.device(cnet.device):
        check(load().pfb_context_split(cnet.data_ptr(), net.data_ptr(), inp.data_ptr(), B, H, W, hidden, context,
                                       dtype_code(cnet.dtype), stream_ptr(cnet.device)), "context_split")
    return net, inp


# ------------------------------------------------------------------------------------------
# encoder-side kernels
# ------------------------------------------------------------------------------------------
def preprocess_frames(images: torch.Tensor, padded_hw, pad_top_left, out_channels: int = 3) -> torch.Tensor:
    """images [B,2,3,H,W] (BGR, [0,1]) -> [2B,Hp,Wp,out_channels] pixel-major RGB in [-1,1] (extra channels zero),
    replicate padded; frame-major."""
    require_cuda(images, "images")
    B, two, three, H, W = images.shape
    if two != 2 or three != 3:
        raise RuntimeError("preprocess_frames: expected images of shape [B,2,3,H,W]")
    Hp, Wp = padded_hw
    out = torch.empty((2 * B, Hp, Wp, out_channels), dtype=images.dtype, device=images.device)
    with torch.cuda.device(images.device):
        check(load().pfb_preprocess_frames(images.data_ptr(), out.data_ptr(), B, H, W, Hp, Wp, pad_top_left[0], pad_top_left[1],
                                           out_channels, dtype_code(images.dtype), stream_ptr(images.device)), "preprocess_frames")
    return out


_inorm_ws = {}
_tls = threading.local()


@contextlib.contextmanager
def scratch_scope(owner: Optional[dict]):
    """While active on this host thread, the small scratch buffers of the normalisation kernels below live in ``owner`` (a dict
    the caller keeps alive) instead of the per-stream cache.  A CUDA graph bakes the addresses of its scratch into its kernels:
    graphs captured on the same stream and replayed concurrently on different ones must not share them, so every capture brings
    its own dict (RAFT._capture)."""
    prev = getattr(_tls, "owner", None)
    _tls.owner = owner
    try:
        yield
    finally:
        _tls.owner = prev


def _scratch(key: tuple, numel: int, device) -> torch.Tensor:
    # per stream in either case: batches in flight on different streams (pipeline.py), the two encoders of one forward on two
    # streams (RAFT._encode); inside a graph the stream is the capture-time one, which is why the owner matters as well
    key = key + (torch.cuda.current_stream(device).cuda_stream,)
    owner = getattr(_tls, "owner", None)
    if owner is None:
        owner = _inorm_ws
    ws = owner.get(key)
    if ws is None:
        ws = owner[key] = torch.empty(numel, dtype=torch.float64, device=device)
    return ws


def instance_norm_act(x: torch.Tensor, relu: bool = True, residual: Optional[torch.Tensor] = None, eps: float = 1e-5,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [B,H,W,C] -> act(IN(x)), or relu(residual + act(IN(x)))."""
    require_cuda(x, "x")
    B, H, W, Cc = x.shape
    y = out if out is not None else torch.empty_like(x)
    ws = _scratch(("inorm", str(x.device), B * Cc), B * Cc * 3, x.device)  # sums (2 doubles) + scale/shift (2 floats)
    if residual is not None:
        require_cuda(residual, "residual")
        assert residual.shape == x.shape
    with torch.cuda.device(x.device):
        check(load().pfb_instance_norm_act(x.data_ptr(), y.data_ptr(), residual.data_ptr() if residual is not None else None,
                                           ws.data_ptr(), B, H, W, Cc, eps, int(relu), dtype_code(x.dtype), stream_ptr(x.device)),
              "instance_norm_act")
    return y


def pack_first_conv(weight: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """weight [64,3,7,7] (fp32, any device) -> the 9 x [128][32] operand tiles of pfb_first_conv7x7s2 (see the header):
    row p*64+co, column 4*t+c of tile j = weight[co, c, j-2p, t-1]; non-swizzled wgmma core-matrix order."""
    co, ci, kh, kw = weight.shape
    if (co, ci, kh, kw) != (64, 3, 7, 7):
        raise RuntimeError("pack_first_conv: expected a [64,3,7,7] filter")
    w = weight.detach().float()
    a = torch.zeros(9, 2, 64, 8, 4, dtype=torch.float32, device=w.device)  # [j][p][co][t][c]
    for j in range(9):
        for p in range(2):
            ky = j - 2 * p
            if 0 <= ky <= 6:
                a[j, p, :, 1:8, :3] = w[:, :, ky, :].permute(0, 2, 1)  # [co][kx][c] -> t = kx + 1
    a = a.reshape(9, 128, 32).to(dtype)
    # [j][row group 16][row 8][K group 4][8 elements] -> [j][row group][K group][row][element]
    return a.reshape(9, 16, 8, 4, 8).permute(0, 1, 3, 2, 4).contiguous()


def pack_flow_conv(weight: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """weight [128,2,7,7] -> the 7 x [128][64] operand tiles of pfb_flow_conv7x7 (see the header)."""
    if tuple(weight.shape) != (128, 2, 7, 7):
        raise RuntimeError("pack_flow_conv: expected a [128,2,7,7] filter")
    w = weight.detach().float()
    a = torch.zeros(7, 128, 8, 8, dtype=torch.float32, device=w.device)  # [ky][co][t][c]
    wk = w.permute(2, 0, 3, 1)  # [ky][co][kx][c]
    a[:, :, 1:8, 0:2] = wk
    a[:, :, 1:8, 2:4] = wk
    a = a.reshape(7, 128, 64).to(dtype)
    # [ky][row group 16][row 8][K group 8][8 elements] -> [ky][row group][K group][row][element]
    return a.reshape(7, 16, 8, 8, 8).permute(0, 1, 3, 2, 4).contiguous()


def flow_conv7x7(flow: torch.Tensor, wpack: torch.Tensor, bias: torch.Tensor, out: torch.Tensor, out_offset: int = 0) -> torch.Tensor:
    """flow fp32 [B,H,W,2] -> out[..., out_offset:out_offset+128] = relu(conv7x7(flow) + bias)."""
    require_cuda(flow, "flow")
    B, H, W, _ = flow.shape
    with torch.cuda.device(flow.device):
        check(load().pfb_flow_conv7x7(flow.data_ptr(), wpack.data_ptr(), bias.data_ptr(), out.data_ptr(), out.shape[-1], out_offset,
                                      B, H, W, dtype_code(out.dtype), stream_ptr(flow.device)), "flow_conv7x7")
    return out


def first_conv7x7s2(x: torch.Tensor, wpack: torch.Tensor, bias: Optional[torch.Tensor], relu: bool,
                    stats_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [N,H,W,4] f16/bf16 -> [N,H/2,W/2,64]; bias fp32 [64] or None; stats_ws: fp64 workspace whose first N*64*2
    entries (zeroed here) receive the per-(image, channel) sums for instance_norm_apply."""
    require_cuda(x, "x")
    N, H, W, C4 = x.shape
    if C4 != 4 or not x.is_contiguous():
        raise RuntimeError("first_conv7x7s2: expected contiguous [N,H,W,4] frames")
    out = torch.empty((N, H // 2, W // 2, 64), dtype=x.dtype, device=x.device)
    if stats_ws is not None:
        stats_ws[: N * 64 * 2].zero_()
    with torch.cuda.device(x.device):
        check(load().pfb_first_conv7x7s2(x.data_ptr(), wpack.data_ptr(), bias.data_ptr() if bias is not None else None, out.data_ptr(),
                                         stats_ws.data_ptr() if stats_ws is not None else None, N, H, W, int(relu), dtype_code(x.dtype),
                                         stream_ptr(x.device)), "first_conv7x7s2")
    return out


def instance_norm_workspace(x_shape, device) -> torch.Tensor:
    B, _, _, Cc = x_shape
    return _scratch(("inorm", str(device), B * Cc), B * Cc * 3, device)  # sums (2 doubles) + scale/shift (2 floats)


def instance_norm_apply(x: torch.Tensor, ws: torch.Tensor, relu: bool = True, residual: Optional[torch.Tensor] = None, eps: float = 1e-5,
                        out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """act(IN(x)) from sums already in ``ws`` (written by first_conv7x7s2)."""
    require_cuda(x, "x")
    B, H, W, Cc = x.shape
    y = out if out is not None else torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(load().pfb_instance_norm_apply(x.data_ptr(), y.data_ptr(), residual.data_ptr() if residual is not None else None,
                                             ws.data_ptr(), B, H, W, Cc, eps, int(relu), dtype_code(x.dtype), stream_ptr(x.device)),
              "instance_norm_apply")
    return y


def bias_act(x: torch.Tensor, bias: Optional[torch.Tensor], relu: bool = True, residual: Optional[torch.Tensor] = None,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [B,H,W,C] -> act(x + bias[c]), or relu(residual + act(x + bias[c])).  bias: fp32 [C] or None."""
    require_cuda(x, "x")
    B, H, W, Cc = x.shape
    y = out if out is not None else torch.empty_like(x)
    ws = _scratch(("bias", str(x.device), Cc), Cc, x.device)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.numel() == Cc and bias.is_cuda
    with torch.cuda.device(x.device):
        check(load().pfb_bias_act(x.data_ptr(), bias.data_ptr() if bias is not None else None,
                                  residual.data_ptr() if residual is not None else None, y.data_ptr(), ws.data_ptr(), B, H, W, Cc,
                                  int(relu), dtype_code(x.dtype), stream_ptr(x.device)), "bias_act")
    return y


# ------------------------------------------------------------------------------------------
# MS-RAFT+ (a17): group norm, the encoders' up-path resize, convex 2x, downflow, scaled on-the-fly lookups
# ------------------------------------------------------------------------------------------
def _opt_f32(t: Optional[torch.Tensor], n: int, name: str):
    if t is None:
        return None
    if t.dtype != torch.float32 or t.numel() != n or not t.is_cuda or not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous fp32 CUDA tensor of {n} elements")
    return t.data_ptr()


def group_norm_act(x: torch.Tensor, gamma: Optional[torch.Tensor], beta: Optional[torch.Tensor], group_size: int,
                   bias: Optional[torch.Tensor] = None, relu: bool = True, residual: Optional[torch.Tensor] = None, eps: float = 1e-5,
                   out: Optional[torch.Tensor] = None, stats_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x [B,H,W,C] -> act(GroupNorm(x + bias)) with ``group_size`` channels per group and the affine gamma / beta (fp32 [C] or
    None), or relu(residual + act(...)).  ``stats_ws``: a workspace whose per-(image, channel) sums of x a producer already
    accumulated (first_conv7x7s2); None computes them here."""
    require_cuda(x, "x")
    B, H, W, Cc = x.shape
    y = out if out is not None else torch.empty_like(x)
    if residual is not None:
        require_cuda(residual, "residual")
        assert residual.shape == x.shape
    args = [_opt_f32(bias, Cc, "bias"), _opt_f32(gamma, Cc, "gamma"), _opt_f32(beta, Cc, "beta"), B, H, W, Cc, group_size, eps, int(relu),
            dtype_code(x.dtype), stream_ptr(x.device)]
    res = residual.data_ptr() if residual is not None else None
    with torch.cuda.device(x.device):
        if stats_ws is None:
            ws = _scratch(("inorm", str(x.device), B * Cc), B * Cc * 3, x.device)
            check(load().pfb_group_norm_act(x.data_ptr(), y.data_ptr(), res, ws.data_ptr(), *args), "group_norm_act")
        else:
            check(load().pfb_group_norm_apply(x.data_ptr(), y.data_ptr(), res, stats_ws.data_ptr(), *args), "group_norm_apply")
    return y


def upsample2x_concat(src: torch.Tensor, skip: Optional[torch.Tensor], out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """src [B,H,W,Cs], skip [B,2H,2W,Ck] -> cat[bilinear 2x (align_corners=False) of src, skip] along the channels."""
    require_cuda(src, "src")
    B, H, W, Cs = src.shape
    Ck = 0 if skip is None else skip.shape[-1]
    if skip is not None:
        require_cuda(skip, "skip")
        if tuple(skip.shape[:3]) != (B, 2 * H, 2 * W) or skip.dtype != src.dtype:
            raise RuntimeError(f"upsample2x_concat: skip {tuple(skip.shape)} does not sit on the 2x grid of src {tuple(src.shape)}")
    if out is None:
        out = torch.empty((B, 2 * H, 2 * W, Cs + Ck), dtype=src.dtype, device=src.device)
    require_cuda(out, "out")
    with torch.cuda.device(src.device):
        check(load().pfb_upsample2x_concat(src.data_ptr(), Cs, skip.data_ptr() if skip is not None else None, Ck, out.data_ptr(), B, H, W,
                                           dtype_code(src.dtype), stream_ptr(src.device)), "upsample2x_concat")
    return out


def convex_upsample2x(coords: torch.Tensor, mask: torch.Tensor, mode: int = 0, out_hw=None, pad=(0, 0)) -> torch.Tensor:
    """coords fp32 [B,H,W,2], mask [B,H,W,36] (x0.25 applied).  mode 0: flow window fp32 [B,2,oh,ow]; mode 1: the upsampled
    absolute coordinates fp32 [B,2H,2W,2] (zero-padded taps)."""
    require_cuda(coords, "coords"); require_cuda(mask, "mask")
    B, H, W, _ = coords.shape
    oh, ow = out_hw or (2 * H, 2 * W)
    shape = (B, 2, oh, ow) if mode == 0 else (B, 2 * H, 2 * W, 2)
    out = torch.empty(shape, dtype=torch.float32, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_convex_upsample2x(coords.data_ptr(), mask.data_ptr(), out.data_ptr(), mode, B, H, W, oh, ow, pad[0], pad[1],
                                           dtype_code(mask.dtype), stream_ptr(coords.device)), "convex_upsample2x")
    return out


def downflow(flow: torch.Tensor, out_hw) -> torch.Tensor:
    """flow fp32 [B,2,H,W] -> bilinear (align_corners=True) [B,2,oh,ow] with u x ow/W, v x oh/H (ms_raft_plus.py:22-35)."""
    require_cuda(flow, "flow")
    B, _, H, W = flow.shape
    out = torch.empty((B, 2) + tuple(out_hw), dtype=torch.float32, device=flow.device)
    with torch.cuda.device(flow.device):
        check(load().pfb_downflow(flow.data_ptr(), out.data_ptr(), B, H, W, out_hw[0], out_hw[1], stream_ptr(flow.device)), "downflow")
    return out


def corr_lookup_onthefly_scaled(fmap1: torch.Tensor, fmap2_pyramid: Sequence[torch.Tensor], coords: torch.Tensor, radius: int, scale: float,
                                tensor_cores: bool, out_stride: Optional[int] = None) -> torch.Tensor:
    """The on-the-fly lookup (pixel-major [B,H,W,out_stride] output) with an explicit scale of the dot products: features stored in
    rows with zero channels beyond their real width C pass 1/sqrt(C).  ``tensor_cores``: the wgmma kernel (+ its SIMT pass for
    flagged queries), else the SIMT kernel."""
    require_cuda(fmap1, "fmap1"); require_cuda(coords, "coords")
    B, H, W, Cc = fmap1.shape
    L = len(fmap2_pyramid)
    planes = L * (2 * radius + 1) ** 2
    stride = (planes + 7) // 8 * 8 if out_stride is None else out_stride
    out = torch.empty((B, H, W, stride), dtype=fmap1.dtype, device=fmap1.device)
    lib = load()
    with torch.cuda.device(fmap1.device):
        if tensor_cores:
            ws = torch.empty(max(1, lib.pfb_corr_lookup_onthefly_tc_workspace_bytes(B, H, W)), dtype=torch.uint8, device=fmap1.device)
            check(lib.pfb_corr_lookup_onthefly_tc_ex(fmap1.data_ptr(), ptr_array(fmap2_pyramid), coords.data_ptr(), out.data_ptr(),
                                                     ws.data_ptr(), B, H, W, Cc, L, radius, scale, dtype_code(fmap1.dtype), stride,
                                                     stream_ptr(fmap1.device)), "corr_lookup_onthefly_tc_ex")
            out._pfb_flags = ws
        else:
            check(lib.pfb_corr_lookup_onthefly_ex(fmap1.data_ptr(), ptr_array(fmap2_pyramid), coords.data_ptr(), out.data_ptr(), B, H, W, Cc,
                                                  L, radius, scale, dtype_code(fmap1.dtype), dtype_code(fmap1.dtype), 0, stride,
                                                  stream_ptr(fmap1.device)), "corr_lookup_onthefly_ex")
    return out


# ------------------------------------------------------------------------------------------
# CCMR (a18): the XCiT block's LayerNorm, LPI convolutions, Fourier features, XCA statistics and fold, upflow2
# ------------------------------------------------------------------------------------------
def layernorm(x: torch.Tensor, gamma: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None, eps: float = 1e-6,
              channels: Optional[int] = None, in_offset: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """LayerNorm over the ``channels`` channels from ``in_offset`` of each pixel of x [..., Cs]; the affine gamma / beta (fp32 [C])
    when given.  Returns [..., C] (or writes ``out``)."""
    require_cuda(x, "x")
    Cs = x.shape[-1]
    Cc = Cs - in_offset if channels is None else channels
    P = x.numel() // Cs
    if out is None:
        out = torch.empty(tuple(x.shape[:-1]) + (Cc,), dtype=x.dtype, device=x.device)
    require_cuda(out, "out")
    with torch.cuda.device(x.device):
        check(load().pfb_layernorm(x.data_ptr(), Cs, in_offset, out.data_ptr(), out.shape[-1], 0, _opt_f32(gamma, Cc, "gamma"),
                                   _opt_f32(beta, Cc, "beta"), P, Cc, eps, dtype_code(x.dtype), stream_ptr(x.device)), "layernorm")
    return out


def depthwise_conv3x3_ex(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, mode: int, addend: Optional[torch.Tensor] = None) -> torch.Tensor:
    """LPI's depthwise 3x3 convolutions (zero padded) of x [B,H,W,C]: mode 0 gelu(dw(x) + bias), mode 1 dw(x) + bias + addend.
    weight fp32 [9, C] tap-major, bias fp32 [C]."""
    require_cuda(x, "x")
    B, H, W, Cc = x.shape
    out = torch.empty_like(x)
    if addend is not None:
        require_cuda(addend, "addend")
    with torch.cuda.device(x.device):
        check(load().pfb_depthwise_conv3x3_ex(x.data_ptr(), Cc, 0, out.data_ptr(), Cc, 0, _opt_f32(weight, 9 * Cc, "weight"),
                                              _opt_f32(bias, Cc, "bias"), addend.data_ptr() if addend is not None else None,
                                              addend.shape[-1] if addend is not None else 0, 0, B, H, W, Cc, mode, dtype_code(x.dtype),
                                              stream_ptr(x.device)), "depthwise_conv3x3_ex")
    return out


def fourier_features(H: int, W: int, dtype: torch.dtype, device) -> torch.Tensor:
    """PositionalEncodingFourier's 64 features before token_projection (xcit.py:73-93): [H, W, 64]."""
    out = torch.empty((H, W, 64), dtype=dtype, device=device)
    with torch.cuda.device(out.device):
        check(load().pfb_fourier_features(out.data_ptr(), H, W, dtype_code(dtype), stream_ptr(out.device)), "fourier_features")
    return out


def xca_stats(qk: torch.Tensor, q_offset: int = 0, k_offset: int = 128) -> torch.Tensor:
    """qk [B,H,W,S] -> fp32 [B, 2304]: per head the 16x16 gram of q, k over the pixels, then the sums of squares of q and of k."""
    require_cuda(qk, "qk")
    B, S = qk.shape[0], qk.shape[-1]
    N = qk.numel() // (B * S)
    lib = load()
    stats = torch.empty((B, 2304), dtype=torch.float32, device=qk.device)
    ws = torch.empty(max(1, lib.pfb_xca_stats_workspace_bytes(B, N)), dtype=torch.uint8, device=qk.device)
    with torch.cuda.device(qk.device):
        check(lib.pfb_xca_stats(qk.data_ptr(), S, q_offset, k_offset, B, N, stats.data_ptr(), ws.data_ptr(), dtype_code(qk.dtype),
                                stream_ptr(qk.device)), "xca_stats")
    return stats


def xca_fold(stats: torch.Tensor, temperature: torch.Tensor, v_w: torch.Tensor, v_b: torch.Tensor, proj_w: torch.Tensor, proj_b: torch.Tensor,
             dtype: torch.dtype):
    """-> (w [B,128 in,128 out], w_k [B*128 out,128 in] or None for fp32, bias fp32 [B,128]) of the folded XCA (pfb_xca_fold)."""
    B = stats.shape[0]
    dev = stats.device
    w = torch.empty((B, 128, 128), dtype=dtype, device=dev)
    wk = torch.empty((B * 128, 128), dtype=dtype, device=dev) if dtype != torch.float32 else None
    bias = torch.empty((B, 128), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(load().pfb_xca_fold(stats.data_ptr(), _opt_f32(temperature, 8, "temperature"), _opt_f32(v_w, 128 * 128, "v_w"),
                                  _opt_f32(v_b, 128, "v_b"), _opt_f32(proj_w, 128 * 128, "proj_w"), _opt_f32(proj_b, 128, "proj_b"),
                                  w.data_ptr(), wk.data_ptr() if wk is not None else None, bias.data_ptr(), B, dtype_code(dtype),
                                  stream_ptr(dev)), "xca_fold")
    return w, wk, bias


def upflow2(flow: torch.Tensor, out_hw=None, pad=(0, 0)) -> torch.Tensor:
    """2 * bilinear 2x (align_corners=True) of flow fp32 [B,2,H,W], the (out_hw, pad) window of the result (ccmr/utils.py:97-99)."""
    require_cuda(flow, "flow")
    B, _, H, W = flow.shape
    oh, ow = out_hw or (2 * H, 2 * W)
    out = torch.empty((B, 2, oh, ow), dtype=torch.float32, device=flow.device)
    with torch.cuda.device(flow.device):
        check(load().pfb_upflow2(flow.data_ptr(), out.data_ptr(), B, H, W, oh, ow, pad[0], pad[1], stream_ptr(flow.device)), "upflow2")
    return out


def convex_handover2x(coords: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """CCMR's handover: fine grid + convex 2x of (coords - grid), coords fp32 [B,H,W,2], mask [B,H,W,36] -> fp32 [B,2H,2W,2]."""
    require_cuda(coords, "coords"); require_cuda(mask, "mask")
    B, H, W, _ = coords.shape
    out = torch.empty((B, 2 * H, 2 * W, 2), dtype=torch.float32, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_convex_handover2x(coords.data_ptr(), mask.data_ptr(), out.data_ptr(), B, H, W, dtype_code(mask.dtype),
                                           stream_ptr(coords.device)), "convex_handover2x")
    return out


# ------------------------------------------------------------------------------------------
# a19: Flow1D
# ------------------------------------------------------------------------------------------
def _pixel_stride(t: torch.Tensor, name: str) -> int:
    """The pixel stride (elements) of a pixel-major [B,H,W,C] view whose pixels are evenly spaced (a channel slice of a wider map)."""
    if not t.is_cuda or t.dim() != 4 or t.stride(3) != 1:
        raise RuntimeError(f"{name} must be a CUDA [B,H,W,C] tensor with unit channel stride")
    B, H, W, _ = t.shape
    s = t.stride(2)
    if (H > 1 and t.stride(1) != W * s) or (B > 1 and t.stride(0) != H * W * s):
        raise RuntimeError(f"{name}: pixels must be evenly spaced (a channel slice of a contiguous [B,H,W,S] map)")
    return s


def attn1d(q: torch.Tensor, k: torch.Tensor, v: Optional[torch.Tensor], axis: int, mode: int = _lib.ATTN1D_ATTN,
           scale: Optional[float] = None, impl: int = 0) -> torch.Tensor:
    """Flow1D's attention / correlation along rows (axis 0) or columns (axis 1) of pixel-major [B,H,W,C] maps (pfb_attn1d).
    mode ATTN1D_ATTN: softmax(scale q k^T) v per sequence -> [B,H,W,C];  ATTN1D_CORR: scale q k^T -> [B*H*W, L] (L = W or H).
    ``scale`` defaults to 1/sqrt(C).  impl: 0 auto (wgmma for f16 / bf16 where the operands qualify), 1 SIMT, 2 wgmma."""
    B, H, W, Cc = q.shape
    if k.shape != q.shape or k.dtype != q.dtype or (v is not None and (v.shape != q.shape or v.dtype != q.dtype)):
        raise RuntimeError("attn1d: q, k (and v) must have equal [B,H,W,C] shapes and dtypes")
    qs, ks = _pixel_stride(q, "q"), _pixel_stride(k, "k")
    vs = _pixel_stride(v, "v") if v is not None else 0
    L = W if axis == 0 else H
    out = torch.empty((B, H, W, Cc) if mode == _lib.ATTN1D_ATTN else (B * H * W, L), dtype=q.dtype, device=q.device)
    os_ = Cc if mode == _lib.ATTN1D_ATTN else L
    with torch.cuda.device(q.device):
        check(load().pfb_attn1d(q.data_ptr(), qs, k.data_ptr(), ks, v.data_ptr() if v is not None else None, vs, out.data_ptr(), os_,
                                B, H, W, Cc, int(axis), int(mode), float(Cc ** -0.5 if scale is None else scale), dtype_code(q.dtype),
                                int(impl), stream_ptr(q.device)), "attn1d")
    return out


def corr1d_lookup(corr_x: torch.Tensor, corr_y: torch.Tensor, coords: torch.Tensor, radius: int,
                  out_stride: Optional[int] = None) -> torch.Tensor:
    """Flow1D's lookup of corr_x [B*H*W, W] and corr_y [B*H*W, H] at coords fp32 [B,H,W,2] -> [B,H,W,out_stride] in the volumes'
    dtype: channels [x taps d = -r..r | y taps d = -r..r], zero beyond 2 (2r+1)."""
    require_cuda(corr_x, "corr_x"); require_cuda(corr_y, "corr_y"); require_cuda(coords, "coords")
    if coords.dtype != torch.float32 or coords.dim() != 4:
        raise RuntimeError("corr1d_lookup: coords must be float32 [B,H,W,2]")
    B, H, W, _ = coords.shape
    if tuple(corr_x.shape) != (B * H * W, W) or tuple(corr_y.shape) != (B * H * W, H) or corr_x.dtype != corr_y.dtype:
        raise RuntimeError("corr1d_lookup: corr_x [B*H*W, W] and corr_y [B*H*W, H] of one dtype")
    stride = 2 * (2 * radius + 1) if out_stride is None else out_stride
    out = torch.empty((B, H, W, stride), dtype=corr_x.dtype, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_corr1d_lookup(corr_x.data_ptr(), corr_y.data_ptr(), coords.data_ptr(), out.data_ptr(), B, H, W, radius,
                                       dtype_code(corr_x.dtype), stride, stream_ptr(coords.device)), "corr1d_lookup")
    return out


# ------------------------------------------------------------------------------------------
# a20: CSFlow
# ------------------------------------------------------------------------------------------
def strip_means(gw: torch.Tensor, gh: torch.Tensor):
    """CSFlow's strip maps of the fmap2 branch (csflow.py:253-260): gw, gh [B,H,W,C] -> (kw [B,1,W,C] column means of gw, kh [B,H,1,C]
    row means of gh), the target grids of the two strip correlations."""
    require_cuda(gw, "gw"); require_cuda(gh, "gh")
    if gw.shape != gh.shape or gw.dtype != gh.dtype or gw.dim() != 4 or not gw.is_contiguous() or not gh.is_contiguous():
        raise RuntimeError("strip_means: gw / gh must be contiguous [B,H,W,C] of one shape and dtype")
    B, H, W, Cc = gw.shape
    kw = torch.empty((B, 1, W, Cc), dtype=gw.dtype, device=gw.device)
    kh = torch.empty((B, H, 1, Cc), dtype=gw.dtype, device=gw.device)
    with torch.cuda.device(gw.device):
        check(load().pfb_strip_means(gw.data_ptr(), gh.data_ptr(), kw.data_ptr(), kh.data_ptr(), B, H, W, Cc, dtype_code(gw.dtype),
                                     stream_ptr(gw.device)), "strip_means")
    return kw, kh


def strip_table_width(n: int, levels: int) -> int:
    """sum over l < levels of n >> l (pfb_strip_table_width)."""
    return sum(n >> l for l in range(levels))


def _ptr_or_none(t: Optional[torch.Tensor]):
    return t.data_ptr() if t is not None else None


def strip_prepare(sw: torch.Tensor, sh: torch.Tensor, grid_hw, levels: int = 4, coords: Optional[torch.Tensor] = None):
    """CSFlow's strip maps sw [B*H*W, W] and sh [B*H*W, H] (any view of that size, e.g. the [Q,1,W] / [Q,H,1] levels of
    corr_volume_build_ex) -> (tab_w fp32 [B*H*W, sum_l W>>l], tab_h fp32 [B*H*W, sum_l H>>l]), the separable strip pyramid.  With
    ``coords`` (fp32 [B,H,W,2]) the initial flow (sum of sh, sum of sw) is added to it in place (csflow.py:176-193)."""
    require_cuda(sw, "sw"); require_cuda(sh, "sh")
    H, W = grid_hw
    Q = sw.numel() // W
    if sw.numel() != Q * W or sh.numel() != Q * H or Q % (H * W) or sw.dtype != sh.dtype or not sw.is_contiguous() or not sh.is_contiguous():
        raise RuntimeError("strip_prepare: sw [B*H*W, W] and sh [B*H*W, H], contiguous, of one dtype")
    if coords is not None and (coords.dtype != torch.float32 or tuple(coords.shape) != (Q // (H * W), H, W, 2) or not coords.is_contiguous()):
        raise RuntimeError("strip_prepare: coords must be contiguous float32 [B,H,W,2]")
    tw = torch.empty((Q, strip_table_width(W, levels)), dtype=torch.float32, device=sw.device)
    th = torch.empty((Q, strip_table_width(H, levels)), dtype=torch.float32, device=sw.device)
    with torch.cuda.device(sw.device):
        check(load().pfb_strip_prepare(sw.data_ptr(), sh.data_ptr(), tw.data_ptr(), th.data_ptr(), _ptr_or_none(coords), Q // (H * W), H, W,
                                       levels, dtype_code(sw.dtype), stream_ptr(sw.device)), "strip_prepare")
    return tw, th


def strip_lookup(tab_w: torch.Tensor, tab_h: torch.Tensor, coords: torch.Tensor, radius: int, levels: int = 4, dtype: torch.dtype = torch.float32,
                 out: Optional[torch.Tensor] = None, out_offset: int = 0) -> torch.Tensor:
    """The strip channel's levels * (2r+1)^2 taps at coords fp32 [B,H,W,2] -> written into ``out`` [B,H,W,S] (a new [B,H,W,planes] tensor
    of ``dtype`` when None) at channels out_offset .., the order of corr_lookup (level, then x offset, then y offset)."""
    require_cuda(coords, "coords")
    if coords.dtype != torch.float32 or coords.dim() != 4 or not coords.is_contiguous():
        raise RuntimeError("strip_lookup: coords must be contiguous float32 [B,H,W,2]")
    B, H, W, _ = coords.shape
    if tab_w.dtype != torch.float32 or tab_h.dtype != torch.float32 or tuple(tab_w.shape) != (B * H * W, strip_table_width(W, levels)) \
            or tuple(tab_h.shape) != (B * H * W, strip_table_width(H, levels)):
        raise RuntimeError("strip_lookup: tab_w / tab_h must be the fp32 tables of strip_prepare for this grid and level count")
    if out is None:
        out = torch.empty((B, H, W, levels * (2 * radius + 1) ** 2), dtype=dtype, device=coords.device)
    if tuple(out.shape[:3]) != (B, H, W) or not out.is_contiguous():
        raise RuntimeError("strip_lookup: out must be contiguous [B,H,W,S]")
    with torch.cuda.device(coords.device):
        check(load().pfb_strip_lookup(tab_w.data_ptr(), tab_h.data_ptr(), coords.data_ptr(), out.data_ptr(), B, H, W, levels, radius,
                                      dtype_code(out.dtype), out.shape[-1], out_offset, stream_ptr(coords.device)), "strip_lookup")
    return out


# ------------------------------------------------------------------------------------------
# a21: SCV
# ------------------------------------------------------------------------------------------
SCV_PLANES = 405  # 5 levels x 9 x 9 bins of the sparse lookup


def knn_topk(f1: torch.Tensor, f2: torch.Tensor, k: int, scale: float = 1.0, impl: int = 0):
    """SCV's k-NN (scv.py:48-83): f1, f2 pixel-major [B,H,W,C] (or [B,N,C]) of one dtype -> (val fp32 [B*N, k] = scale * <f1[q], f2[t]>,
    idx int32 [B*N, k] = t, the target pixel within its sample), the k largest scores of each query, descending, ties to the lower
    target.  1 <= k <= 32, k <= N.  impl 0: wgmma where the operands qualify (f16 / bf16, C a multiple of 64 up to 256), SIMT
    otherwise; 1: SIMT; 2: wgmma or an error."""
    require_cuda(f1, "f1"); require_cuda(f2, "f2")
    if f1.shape != f2.shape or f1.dtype != f2.dtype or f1.dim() not in (3, 4) or not f1.is_contiguous() or not f2.is_contiguous():
        raise RuntimeError("knn_topk: f1 / f2 must be contiguous pixel-major tensors of one shape and dtype")
    B, Cc = f1.shape[0], f1.shape[-1]
    N = f1[0].numel() // Cc
    val = torch.empty((B * N, k), dtype=torch.float32, device=f1.device)
    idx = torch.empty((B * N, k), dtype=torch.int32, device=f1.device)
    lib, dt = load(), dtype_code(f1.dtype)
    with torch.cuda.device(f1.device):
        nbytes = lib.pfb_knn_topk_workspace_bytes(f1.data_ptr(), f2.data_ptr(), B, N, Cc, k, dt, impl)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=f1.device) if nbytes else None
        check(lib.pfb_knn_topk(f1.data_ptr(), f2.data_ptr(), val.data_ptr(), idx.data_ptr(), _ptr_or_none(ws), nbytes, B, N, Cc, k,
                               float(scale), dt, impl, stream_ptr(f1.device)), "knn_topk")
    return val, idx


def sparse_prepare(val: torch.Tensor, idx: torch.Tensor, coords: torch.Tensor) -> torch.Tensor:
    """(val, idx) of knn_topk on the grid of coords (fp32 [B,H,W,2], after the warm start) -> the fp32 table [B*H*W, k, 3] of
    (ty + wy, tx + wx, val), w = coords - grid."""
    require_cuda(val, "val"); require_cuda(idx, "idx"); require_cuda(coords, "coords")
    if coords.dtype != torch.float32 or coords.dim() != 4 or not coords.is_contiguous():
        raise RuntimeError("sparse_prepare: coords must be contiguous float32 [B,H,W,2]")
    B, H, W, _ = coords.shape
    k = val.shape[-1]
    if val.dtype != torch.float32 or idx.dtype != torch.int32 or tuple(val.shape) != (B * H * W, k) or tuple(idx.shape) != (B * H * W, k) \
            or not val.is_contiguous() or not idx.is_contiguous():
        raise RuntimeError("sparse_prepare: val fp32 and idx int32 [B*H*W, k], contiguous")
    table = torch.empty((B * H * W, k, 3), dtype=torch.float32, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_sparse_prepare(val.data_ptr(), idx.data_ptr(), coords.data_ptr(), table.data_ptr(), B, H, W, k,
                                        stream_ptr(coords.device)), "sparse_prepare")
    return table


def sparse_lookup(table: torch.Tensor, coords: torch.Tensor, dtype: torch.dtype = torch.float32,
                  out_stride: Optional[int] = None) -> torch.Tensor:
    """SCV's per-iteration lookup (scv.py:248-298) at coords fp32 [B,H,W,2] -> [B,H,W,out_stride] of ``dtype``: the 405 bins (level, then
    y offset, then x offset), zero beyond."""
    require_cuda(table, "table"); require_cuda(coords, "coords")
    if coords.dtype != torch.float32 or coords.dim() != 4 or not coords.is_contiguous():
        raise RuntimeError("sparse_lookup: coords must be contiguous float32 [B,H,W,2]")
    B, H, W, _ = coords.shape
    if table.dtype != torch.float32 or table.dim() != 3 or table.shape[0] != B * H * W or table.shape[2] != 3 or not table.is_contiguous():
        raise RuntimeError("sparse_lookup: table must be the contiguous fp32 [B*H*W, k, 3] of sparse_prepare")
    stride = SCV_PLANES if out_stride is None else out_stride
    out = torch.empty((B, H, W, stride), dtype=dtype, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_sparse_lookup(table.data_ptr(), coords.data_ptr(), out.data_ptr(), B, H, W, table.shape[1], dtype_code(dtype), stride,
                                       stream_ptr(coords.device)), "sparse_lookup")
    return out


def convex_upsample4x(coords: torch.Tensor, mask: torch.Tensor, out_hw=None, pad=(0, 0)):
    """coords fp32 [B,H,W,2], mask [B,H,W,144] -> (flow_up fp32 [B,2,oh,ow] of the convex 4x of 4 * flow, flow_small fp32 [B,2,H,W])
    (scv.py:186-197)."""
    require_cuda(coords, "coords"); require_cuda(mask, "mask")
    B, H, W, _ = coords.shape
    oh, ow = out_hw or (4 * H, 4 * W)
    up = torch.empty((B, 2, oh, ow), dtype=torch.float32, device=coords.device)
    small = torch.empty((B, 2, H, W), dtype=torch.float32, device=coords.device)
    with torch.cuda.device(coords.device):
        check(load().pfb_convex_upsample4x(coords.data_ptr(), mask.data_ptr(), up.data_ptr(), small.data_ptr(), B, H, W, oh, ow,
                                           pad[0], pad[1], dtype_code(mask.dtype), stream_ptr(coords.device)), "convex_upsample4x")
    return up, small


# ------------------------------------------------------------------------------------------
# a22: LLA-Flow
# ------------------------------------------------------------------------------------------
LLA_TAPS, LLA_K = 25, 26 * 256  # the 5 x 5 local window; K of the shifted volume GEMM


def local_similar(qk: torch.Tensor):
    """qk [B,H,W,512] = [q1 | k1 | q2 | k2] -> (a1, a2) fp32 [B*H*W, 25]: softmax over the 5 x 5 clamped window of <q, k> / sqrt(128)."""
    require_cuda(qk, "qk")
    B, H, W, Cc = qk.shape
    if Cc != 512:
        raise RuntimeError(f"local_similar: qk must have 512 channels ([q1 | k1 | q2 | k2]), got {Cc}")
    a1 = torch.empty((B * H * W, LLA_TAPS), dtype=torch.float32, device=qk.device)
    a2 = torch.empty_like(a1)
    with torch.cuda.device(qk.device):
        check(load().pfb_local_similar(qk.data_ptr(), a1.data_ptr(), a2.data_ptr(), B, H, W, dtype_code(qk.dtype), stream_ptr(qk.device)),
              "local_similar")
    return a1, a2


def _lla_check(name: str, *ts: torch.Tensor) -> None:
    for i, t in enumerate(ts):
        require_cuda(t, f"{name} arg {i}")
        if t.shape != ts[0].shape or t.dtype != ts[0].dtype or t.dim() != 4 or t.shape[-1] != 256:
            raise RuntimeError(f"{name}: features must be [B,H,W,256] of one shape and dtype")


def local_aggregate(fmap2: torch.Tensor, v: torch.Tensor, a2: torch.Tensor, gamma: float) -> torch.Tensor:
    """fmap2 + gamma * sum_l a2[:, l] v[clamp(n + delta_l)] -> [B,H,W,256] in the storage type."""
    _lla_check("local_aggregate", fmap2, v)
    require_cuda(a2, "a2")
    B, H, W, _ = fmap2.shape
    out = torch.empty_like(fmap2)
    with torch.cuda.device(fmap2.device):
        check(load().pfb_local_aggregate(fmap2.data_ptr(), v.data_ptr(), a2.data_ptr(), float(gamma), out.data_ptr(), B, H, W,
                                         dtype_code(fmap2.dtype), stream_ptr(fmap2.device)), "local_aggregate")
    return out


def shift_pack(fmap1: torch.Tensor, f1: torch.Tensor, a1: torch.Tensor, fmap2p: torch.Tensor, f2: torch.Tensor, gamma: float,
               padded: bool = True):
    """The shifted volume's operands: (A' [B,H,W,6656], [fmap2' | f2''] replicate-padded [B,H+4,W+4,512]) when ``padded``, else
    (A', B' [B,H,W,6656])."""
    _lla_check("shift_pack", fmap1, f1, fmap2p, f2)
    require_cuda(a1, "a1")
    B, H, W, _ = fmap1.shape
    a = torch.empty((B, H, W, LLA_K), dtype=fmap1.dtype, device=fmap1.device)
    b = torch.empty((B, H + 4, W + 4, 512) if padded else (B, H, W, LLA_K), dtype=fmap1.dtype, device=fmap1.device)
    with torch.cuda.device(fmap1.device):
        check(load().pfb_shift_pack(fmap1.data_ptr(), f1.data_ptr(), a1.data_ptr(), fmap2p.data_ptr(), f2.data_ptr(), float(gamma),
                                    a.data_ptr(), b.data_ptr() if padded else None, None if padded else b.data_ptr(), B, H, W,
                                    dtype_code(fmap1.dtype), stream_ptr(fmap1.device)), "shift_pack")
    return a, b


def shift_volume_tiled(a_pack: torch.Tensor, b_pad: torch.Tensor, levels: int = 4) -> List[torch.Tensor]:
    """A' [B,H,W,6656], padded [fmap2' | f2''] [B,H+4,W+4,512] (f16 / bf16) -> the tiled pyramid of <A'[n], B'[m]> (as
    corr_volume_build_tiled returns it)."""
    require_cuda(a_pack, "a_pack"); require_cuda(b_pad, "b_pad")
    B, H, W, K = a_pack.shape
    if K != LLA_K or tuple(b_pad.shape) != (B, H + 4, W + 4, 512) or b_pad.dtype != a_pack.dtype:
        raise RuntimeError("shift_volume_tiled: a_pack [B,H,W,6656] and b_pad [B,H+4,W+4,512] of one dtype")
    lib = load()
    pyr = []
    for l in range(levels):
        nbytes = lib.pfb_corr_level_bytes_tiled(B, H, W, H, W, l)
        if nbytes == 0:
            raise RuntimeError(f"shift_volume_tiled: {H}x{W} grid too small for {levels} levels")
        pyr.append(torch.empty((B * H * W, nbytes // (2 * B * H * W)), dtype=a_pack.dtype, device=a_pack.device))
    with torch.cuda.device(a_pack.device):
        check(lib.pfb_shift_volume_tiled(a_pack.data_ptr(), b_pad.data_ptr(), ptr_array(pyr), B, H, W, levels, dtype_code(a_pack.dtype),
                                         stream_ptr(a_pack.device)), "shift_volume_tiled")
    return pyr
