"""CSFlow (cross-strip correlation) on libptlflow_b200.

Surface kept from ptlflow/models/csflow/csflow.py:38-224: class name ``csflow``, the constructor keywords (``corr_levels, corr_radius,
dropout, gamma, max_flow, iters, gen_fmap, skip_encode``), the checkpoint table, the state_dict keys (``fnet.*``, ``cnet.*`` as RAFT's
BasicEncoder, ``strip_corr_block_v2.conv{1_1,1_2,2_1,2_2}.{conv,bn}.*``, ``update_block.*`` as RAFT's BasicUpdateBlock with
``encoder.convc1`` over 2 L (2r+1)^2 channels), ``forward(dict) -> dict`` with ``flows`` [B,1,2,H,W] and ``flow_small`` [B,2,H/8,W/8],
and the warm start from ``prev_preds.flow_small``.

Kernel mapping (DESIGN.md section 1, row a20): the encoders, pre-processing, CUDA-graph capture, warm start and RAFT's 4D pyramid are
RAFT's.  CSFlowEngine adds the strip module: its four ConvBNReLU 1x1 convolutions on the wgmma (f16 / bf16) or SIMT (fp32)
convolution, pfb_strip_means, the two strip correlations on pfb_corr_volume_build_ex, and pfb_strip_prepare, which stores the strip
channel's pyramid as separable fp32 tables and adds the initial strip flow to the coordinates.  The loop is pfb_raft_refine with variant
PFB_VARIANT_CSFLOW (8), whose lookup is RAFT's followed by pfb_strip_lookup.
"""
from __future__ import annotations

from typing import Dict

import torch.nn as nn

from ... import _lib
from ...engine import CSFlowEngine
from ...utils.registry import register_model, trainable
from ..raft.extractor import BasicEncoder
from ..raft.raft import RAFT
from ..raft.update import BasicUpdateBlock, _no_forward


class ConvBNReLU(nn.Module):
    """Parameter container of csflow.py:299-319 (1x1 convolution without bias, BatchNorm, ReLU); CSFlowEngine folds it."""

    def __init__(self, in_chan: int, out_chan: int) -> None:
        super().__init__()
        self.conv = nn.Conv2d(in_chan, out_chan, kernel_size=1, bias=False)
        self.bn = nn.BatchNorm2d(out_chan)
        nn.init.kaiming_normal_(self.conv.weight, a=1)

    forward = _no_forward


class StripCrossCorrMap_v2(nn.Module):
    """Parameter container of csflow.py:227-237: f1w / f1h from fmap1 (conv1_1 / conv1_2), the strips of fmap2 (conv2_1 / conv2_2)."""

    def __init__(self, in_chan: int = 256, out_chan: int = 256) -> None:
        super().__init__()
        self.conv1_1 = ConvBNReLU(in_chan, out_chan)
        self.conv1_2 = ConvBNReLU(in_chan, out_chan)
        self.conv2_1 = ConvBNReLU(in_chan, out_chan)
        self.conv2_2 = ConvBNReLU(in_chan, out_chan)

    forward = _no_forward


class CSFlow(RAFT):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/csflow-chairs-458a9436.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/csflow-things-ebdd403b.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/csflow-kitti-dc66357a.ckpt",
    }
    _variant = _lib.VARIANT_CSFLOW
    _engine_cls = CSFlowEngine
    min_grid = 16  # 1/8-resolution pixels per side: the coarsest of the 4 levels keeps 2, below that the reference divides by 0

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, gen_fmap: bool = False, skip_encode: bool = False, **kwargs) -> None:
        if corr_levels != 4:
            # CSFlow.forward builds a 4-level pyramid whatever corr_levels says (csflow.py:158, 448), while convc1 is sized from it
            raise ValueError(f"csflow's pyramid always has 4 levels (the reference fails with any other corr_levels), got {corr_levels}")
        if not 0 <= corr_radius <= 15:
            raise ValueError(f"csflow's lookup supports corr_radius 0..15, got {corr_radius}")
        if gen_fmap or skip_encode:
            raise ValueError("csflow: gen_fmap and skip_encode (the reference's debugging paths) are not supported")
        if iters < 1:
            raise ValueError(f"csflow needs at least one iteration (the convex upsample reads the last mask), got iters={iters}")
        self.gen_fmap, self.skip_encode = gen_fmap, skip_encode
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow, iters=iters,
                         alternate_corr=False, **kwargs)
        self.has_trained_on_ptlflow = False

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        self.fnet = BasicEncoder(output_dim=256, norm_fn="instance", dropout=self.dropout)
        self.cnet = BasicEncoder(output_dim=self.hidden_dim + self.context_dim, norm_fn="batch", dropout=self.dropout)
        self.strip_corr_block_v2 = StripCrossCorrMap_v2(in_chan=256, out_chan=256)
        # BasicMotionEncoder_v2 (csflow.py:654-665): RAFT's motion encoder over twice the lookup planes, 2 L (2r+1)^2
        self.update_block = BasicUpdateBlock(2 * self.corr_levels, self.corr_radius, hidden_dim=self.hidden_dim)

    def _loop_parameters(self):
        return list(self.update_block.parameters()) + list(self.strip_corr_block_v2.parameters())

    def _extra_engine_args(self) -> Dict:
        return {"strip_block": self.strip_corr_block_v2}

    def _check_grid(self, h8: int, w8: int) -> None:
        # bilinear_sampler normalises by (W_l - 1) and (H_l - 1) of every level (csflow.py:506-511): a coarsest level of one pixel
        # makes the reference return NaN
        if min(h8, w8) < self.min_grid:
            raise ValueError(f"csflow needs a 1/8-resolution grid of at least {self.min_grid} pixels per side (images of more than "
                             f"{8 * (self.min_grid - 1)} px after padding); got {h8} x {w8}")


@register_model
@trainable
class csflow(CSFlow):
    pass
