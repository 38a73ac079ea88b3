"""Flow1D (1D cross-attention and row / column correlation) on libptlflow_b200.

Surface kept from ptlflow/models/flow1d/flow1d.py:45-252: class name ``flow1d``, the constructor keywords (``downsample_factor,
feature_channels, hidden_dim, context_dim, corr_radius, iters, mixed_precision, gamma, max_flow``), the checkpoint table, the
state_dict keys (``fnet.*``, ``cnet.*`` as RAFT's BasicEncoder, ``attn_x.*`` / ``attn_y.*`` with their ``self_attn``, and
``update_block.*`` as RAFT's BasicUpdateBlock with ``encoder.convc1`` over 2 (2r+1) channels), ``forward(dict) -> dict`` with
``flows`` [B,1,2,H,W] and ``flow_small`` [B,2,H/8,W/8], and the warm start from ``prev_preds.flow_small``.

Kernel mapping (DESIGN.md section 1, row a19): the encoders, pre-processing, CUDA-graph capture and warm start are RAFT's.  The
correlation pyramid is replaced by Flow1DEngine.build_volume: the attentions' 1x1 query / key projections on the wgmma (f16 / bf16)
or SIMT (fp32) convolution, four pfb_attn1d attentions and two pfb_attn1d correlations, which store a row volume [B*H*W, W] and a
column volume [B*H*W, H].  The loop is pfb_raft_refine with variant PFB_VARIANT_FLOW1D (7), whose lookup is pfb_corr1d_lookup.
"""
from __future__ import annotations

from typing import Dict

import torch.nn as nn

from ... import _lib
from ...engine import Flow1DEngine
from ...utils.registry import register_model, trainable
from ..raft.extractor import BasicEncoder
from ..raft.raft import RAFT
from ..raft.update import BasicUpdateBlock, _no_forward


class Attention1D(nn.Module):
    """Parameter container of attention.py:6-38 (query / key 1x1 convolutions with bias; with ``double_cross_attn`` a self-attention
    along the other axis first); Flow1DEngine packs it."""

    def __init__(self, in_channels: int, y_attention: bool = False, double_cross_attn: bool = False) -> None:
        super().__init__()
        self.y_attention = y_attention
        if double_cross_attn:
            self.self_attn = Attention1D(in_channels, y_attention=not y_attention)
        self.query_conv = nn.Conv2d(in_channels, in_channels, 1)
        self.key_conv = nn.Conv2d(in_channels, in_channels, 1)
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    forward = _no_forward


class Flow1D(RAFT):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/flow1d-chairs-75cd85a1.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/flow1d-things-bcd92815.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/flow1d-sintel-28a093d3.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/flow1d-kitti-803a0181.ckpt",
        "highres": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/flow1d-highres-7ab476dc.ckpt",
    }
    _variant = _lib.VARIANT_FLOW1D
    _engine_cls = Flow1DEngine

    def __init__(self, downsample_factor: int = 8, feature_channels: int = 256, hidden_dim: int = 128, context_dim: int = 128,
                 corr_radius: int = 32, iters: int = 32, mixed_precision: bool = False, gamma: float = 0.8, max_flow: float = 400,
                 **kwargs) -> None:
        if downsample_factor != 8:
            raise ValueError(f"flow1d runs at 1/8 resolution only (downsample_factor=8), got {downsample_factor}")
        if hidden_dim != 128 or context_dim != 128:
            raise ValueError(f"flow1d's update block runs hidden_dim = context_dim = 128, got {hidden_dim} / {context_dim}")
        if feature_channels <= 0 or feature_channels % 64 != 0 or feature_channels > 256:
            raise ValueError(f"flow1d's 1D attention needs feature_channels a multiple of 64, at most 256; got {feature_channels}")
        if not 1 <= corr_radius <= 64:
            raise ValueError(f"flow1d's 1D lookup supports corr_radius 1..64, got {corr_radius}")
        if iters < 1:
            raise ValueError(f"flow1d needs at least one iteration (the convex upsample reads the last mask), got iters={iters}")
        self.downsample_factor, self.feature_channels, self.mixed_precision = downsample_factor, feature_channels, mixed_precision
        super().__init__(corr_levels=1, corr_radius=corr_radius, gamma=gamma, max_flow=max_flow, iters=iters, alternate_corr=False,
                         **kwargs)
        self.has_trained_on_ptlflow = False

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        C = self.feature_channels
        self.fnet = BasicEncoder(output_dim=C, norm_fn="instance", dropout=0.0)
        self.cnet = BasicEncoder(output_dim=self.hidden_dim + self.context_dim, norm_fn="batch", dropout=0.0)
        self.attn_x = Attention1D(C, y_attention=False, double_cross_attn=True)
        self.attn_y = Attention1D(C, y_attention=True, double_cross_attn=True)
        self.update_block = BasicUpdateBlock(1, 0, hidden_dim=self.hidden_dim)
        self.update_block.encoder.convc1 = nn.Conv2d(2 * (2 * self.corr_radius + 1), 256, 1)  # [corr_x | corr_y] taps

    def _loop_parameters(self):
        return list(self.update_block.parameters()) + list(self.attn_x.parameters()) + list(self.attn_y.parameters())

    def _extra_engine_args(self) -> Dict:
        return {"attention": (self.attn_x, self.attn_y)}

    def _check_grid(self, h8: int, w8: int) -> None:
        # the sample positions are normalised by W8 - 1 and H8 - 1 (correlation.py:41, 66); one sequence holds a row or a column
        if min(h8, w8) < 2 or max(h8, w8) > _lib.ATTN1D_MAX_L:
            raise ValueError(f"flow1d needs a 1/8-resolution grid of 2 .. {_lib.ATTN1D_MAX_L} pixels per side (images of 9 .. "
                             f"{8 * _lib.ATTN1D_MAX_L} px after padding); got {h8} x {w8}")


@register_model
@trainable
class flow1d(Flow1D):
    pass
