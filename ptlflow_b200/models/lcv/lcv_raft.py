"""LCV (learnable cost volume, Cayley representation) on RAFT's and raft_small's refinement loops, on libptlflow_b200.

Surface kept from ptlflow/models/lcv/lcv_raft.py:41-235: class names ``lcv_raft`` / ``lcv_raft_small``, the constructor keywords
(``corr_levels, corr_radius, dropout, gamma, max_flow, iters``; there is no ``alternate_corr``), the checkpoint tables, the state_dict
keys (RAFT's / raft_small's plus ``corr_block.raw_P`` [C,C], ``corr_block.raw_D`` [C] and the persistent buffer ``corr_block.eye``),
``forward(dict) -> dict`` with ``flows`` [B,1,2,H,W] and ``flow_small`` [B,2,H/8,W/8], and the warm start from
``prev_preds.flow_small``.

Kernel mapping (DESIGN.md section 1, row a25): encoders, CUDA-graph capture, warm start, update blocks and upsampling are RAFT's /
raft_small's, and the loop is pfb_raft_refine with VARIANT_RAFT / VARIANT_RAFT_SMALL.  LCVEngine folds W / sqrt(C) of the
LearnableCorrBlock in fp64 and applies it to fmap1 as a 1x1 convolution (wgmma in f16 / bf16, SIMT in fp32); the volume builders
make the distinct levels of corr_lcv.py:44-50's pyramid, which stops pooling once a level's smaller side is <= 2r+1, and the lookup
reads the repeated levels at their own size (pfb_raft_buffers.pool_min_side, pfb_corr_level_sizes).

Unlike RAFT, the reference feeds the encoders BGR frames (lcv_raft.py:126-134, bgr_to_rgb=False); the shared pre-processing
kernel writes RGB, so both encoders' first convolutions run with their input channels reversed, which is the same arithmetic.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict

import torch
import torch.nn as nn

from ...engine import LCVEngine
from ...utils.registry import ptlflow_trained, register_model, trainable
from ..raft.extractor import BasicEncoder, SmallEncoder
from ..raft.raft import RAFT, RAFTSmall
from ..raft.update import _no_forward


class LearnableCorrBlock(nn.Module):
    """Parameter container of corr_lcv.py:8-17 (raw_P = I, raw_D = 0 and the ``eye`` buffer, as the reference initialises them);
    LCVEngine folds them into W."""

    def __init__(self, dim: int, num_levels: int = 4, radius: int = 4) -> None:
        super().__init__()
        self.num_levels, self.radius, self.dim = num_levels, radius, dim
        self.raw_P = nn.Parameter(torch.eye(dim), requires_grad=True)
        self.raw_D = nn.Parameter(torch.zeros(dim), requires_grad=True)
        self.register_buffer("eye", torch.eye(dim))

    forward = _no_forward


class _BgrInput:
    """An encoder whose frames arrive RGB but whose weights expect BGR: its first convolution is planned with the input channels
    reversed (the pre-processing treats the three channels alike, so this equals feeding it BGR)."""

    def _layers(self):
        (conv1, norm1), blocks, proj = super()._layers()
        keep = ("kernel_size", "stride", "padding", "dilation", "groups", "padding_mode", "in_channels", "out_channels", "bias")
        bgr = SimpleNamespace(**{k: getattr(conv1, k) for k in keep}, weight=conv1.weight.detach().flip(1))
        return (bgr, norm1), blocks, proj


class _BgrBasicEncoder(_BgrInput, BasicEncoder):
    pass


class _BgrSmallEncoder(_BgrInput, SmallEncoder):
    pass


class _LCV:
    """What LCV adds to RAFT / RAFTSmall (put in front of either): the learned volume's engine and corr_block, encoders that take BGR
    frames, and the reference's constructor keywords without ``alternate_corr``."""

    _engine_cls = LCVEngine

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, **kwargs) -> None:
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow, iters=iters,
                         alternate_corr=False, **kwargs)
        if hasattr(self.hparams, "alternate_corr"):  # collected from RAFT's constructor; LCV has no on-the-fly mode
            delattr(self.hparams, "alternate_corr")

    def _build_networks(self) -> None:
        super()._build_networks()
        self.corr_block = LearnableCorrBlock(self.fnet.conv2.out_channels, self.corr_levels, self.corr_radius)

    def _loop_parameters(self):
        # W is folded from raw_P, raw_D and eye: a reloaded or edited checkpoint is folded again
        return list(self.update_block.parameters()) + list(self.corr_block.parameters()) + list(self.corr_block.buffers())

    def _extra_engine_args(self) -> Dict:
        return {"corr_block": self.corr_block}


class LCV_RAFT(_LCV, RAFT):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/lcv_raft-chairs-8063d698.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/lcv_raft-things-4c7233b8.ckpt",
    }
    _encoder_cls = _BgrBasicEncoder


class LCV_RAFTSmall(_LCV, RAFTSmall):
    pretrained_checkpoints = {}
    _encoder_cls = _BgrSmallEncoder

    def __init__(self, corr_levels: int = 4, corr_radius: int = 3, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, **kwargs) -> None:
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow, iters=iters,
                         **kwargs)


@register_model
@trainable
@ptlflow_trained
class lcv_raft(LCV_RAFT):
    pass


@register_model
@trainable
@ptlflow_trained
class lcv_raft_small(LCV_RAFTSmall):
    pass
