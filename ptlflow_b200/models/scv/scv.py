"""SCV (sparse cost volume, Jiang et al., CVPR 2021) on libptlflow_b200.

Surface kept from ptlflow/models/scv/scv.py:112-512: the registered names ``scv4`` (SCVQuarter: 1/4-resolution loop, convex 4x) and
``scv8`` (SCVEighth: 1/8, convex 8x), the constructor keywords (``num_k, gamma, max_flow, iters``), the checkpoint tables, the
state_dict keys (``fnet.*`` / ``cnet.*`` as the reference's encoders, whose residual blocks all carry a 1x1 projection shortcut,
``update_block.*`` as RAFT's BasicUpdateBlock with ``encoder.convc1`` over 405 channels and, for scv4, a 144-channel ``mask.2``),
``forward(dict) -> dict`` with ``flows`` [B,1,2,H,W] and ``flow_small`` at the loop's grid, and the warm start from
``prev_preds.flow_small``.  Neither faiss nor torch_scatter is needed.

Kernel mapping (DESIGN.md section 1, row a21): the encoders, pre-processing, CUDA-graph capture and warm start are RAFT's.  SCVEngine
keeps the num_k best matches of every query with pfb_knn_topk (the all-pairs volume is never materialised), folds them and the warm
start into a per-query table with pfb_sparse_prepare, and runs pfb_raft_refine with variant PFB_VARIANT_SCV8 / PFB_VARIANT_SCV4,
whose lookup is pfb_sparse_lookup.
"""
from __future__ import annotations

from typing import Dict

import torch.nn as nn

from ... import _lib
from ...engine import SCVEngine
from ...utils.registry import register_model, trainable
from ..raft.extractor import BasicEncoder
from ..raft.raft import RAFT
from ..raft.update import BasicUpdateBlock

MAX_K = 32  # pfb_knn_topk keeps at most 32 matches per query


class SCVEncoder(BasicEncoder):
    """BasicEncoder of scv/extractor.py:122-195: every ResidualBlock has a 1x1 convolution + norm shortcut, stride 1 included."""

    project_shortcut = True


class SCVEncoderQuarter(SCVEncoder):
    """BasicEncoderQuarter of scv/extractor.py:197-270: stage strides 1, 2, 1, output at 1/4."""

    strides = (1, 2, 1)


class SCVBase(RAFT):
    _engine_cls = SCVEngine
    _encoder_cls = SCVEncoder
    _mask_channels = 576
    grid_stride = 8  # image pixels per loop-grid pixel

    def __init__(self, num_k: int = 32, gamma: float = 0.8, max_flow: float = 400, iters: int = 32, **kwargs) -> None:
        if iters < 1:
            raise ValueError(f"scv needs at least one iteration (the convex upsample reads the last mask), got iters={iters}")
        self.num_k = num_k
        # 5 levels of 9 x 9 bins (scv.py:245-260): convc1 sees 405 planes, as RAFT's update block with corr_levels 5, radius 4
        super().__init__(corr_levels=5, corr_radius=4, dropout=0.0, gamma=gamma, max_flow=max_flow, iters=iters, alternate_corr=False,
                         **kwargs)
        self.has_trained_on_ptlflow = False

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        self.fnet = self._encoder_cls(output_dim=256, norm_fn="instance", dropout=0.0)
        self.cnet = self._encoder_cls(output_dim=256, norm_fn="batch", dropout=0.0)
        self.update_block = BasicUpdateBlock(self.corr_levels, self.corr_radius, hidden_dim=self.hidden_dim)
        if self._mask_channels != 576:
            self.update_block.mask[2] = nn.Conv2d(256, self._mask_channels, 1)

    @property
    def num_k(self) -> int:
        return self.__dict__["_num_k"]

    @num_k.setter
    def num_k(self, value: int) -> None:
        if not 1 <= value <= MAX_K:
            raise ValueError(f"scv keeps 1..{MAX_K} matches per query, got num_k={value}")
        self.__dict__["_num_k"] = int(value)

    def _extra_engine_args(self) -> Dict:
        return {"num_k": self.num_k}

    def _get_engine(self, dtype, device):
        if self._engine is not None and self._engine.num_k != self.num_k:
            self._engine = None  # the engine was built for another num_k
        return super()._get_engine(dtype, device)

    def _graph_key(self, images, flow_init) -> tuple:
        return super()._graph_key(images, flow_init) + (self.num_k,)

    def _check_grid(self, h8: int, w8: int) -> None:
        f = 8 // self.grid_stride
        if h8 * w8 * f * f < self.num_k:
            raise ValueError(f"scv keeps num_k={self.num_k} matches per query, but the {h8 * f} x {w8 * f} grid of the padded images has "
                             f"fewer pixels")


class SCVQuarter(SCVBase):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/scv-quarter-chairs-4726627e.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/scv-quarter-kitti-e86c7953.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/scv-quarter-sintel-2d9b4a05.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/scv-quarter-things-0dac9b66.ckpt",
    }
    _variant = _lib.VARIANT_SCV4
    _encoder_cls = SCVEncoderQuarter
    _mask_channels = 144  # 9 taps x 4 x 4 (scv/update.py:161-165)
    grid_stride = 4


class SCVEighth(SCVBase):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/scv-eighth-chairs-8ba57294.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/scv-eighth-things-9c893323.ckpt",
    }
    _variant = _lib.VARIANT_SCV8


@register_model
@trainable
class scv4(SCVQuarter):
    pass


@register_model
@trainable
class scv8(SCVEighth):
    pass
