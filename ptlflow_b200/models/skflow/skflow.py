"""SKFlow (large-kernel update block on the GMA loop) on libptlflow_b200.

Surface kept from ptlflow/models/skflow/skflow.py:51-232: class name ``skflow``, constructor keywords (``corr_levels,
corr_radius, dropout, gamma, max_flow, iters, k_conv, PCUpdater_conv, num_heads, position_only, position_and_content,
alternate_corr``), state_dict keys (``fnet.*, cnet.*, update_block.{encoder,gru,flow_head,mask,aggregator}.*, att.*`` with the
PCBlocks' ``conv_list.N / ffn1.0 / ffn1.2 / pw / ffn2.0 / ffn2.2``), ``forward(dict) -> dict`` with ``flows`` and ``flow_small``
and the ``prev_preds.flow_small`` warm start.

Kernel mapping (DESIGN.md section 1, row a15): the encoders, the correlation volume / lookup, the attention and its
aggregate are GMA's.  Each PCBlock4_Deep_nopool_res (update.py:7-41) is five 1x1 convolutions on the implicit-GEMM kernels
(GELU and residual + GELU epilogues; a leading k = 1 entry of k_conv rides the ffn1 epilogue) and one fused depthwise
convolution + residual + GELU kernel per other entry of k_conv; the whole loop runs in pfb_skflow_refine (ptlflow_b200/engine.py
SKFlowEngine).
"""
from __future__ import annotations

from typing import Sequence

import torch.nn as nn

from ... import _lib
from ...engine import SKFlowEngine
from ...utils.registry import register_model, trainable
from ..gma.gma import GMA, Aggregate, Attention
from ..raft.extractor import BasicEncoder
from ..raft.update import _no_forward


class PCBlock4_Deep_nopool_res(nn.Module):
    """Parameter container of update.py:7-41: depthwise k x k convolutions ``conv_list``, FFNs ``ffn1`` / ``ffn2`` (1x1, GELU,
    1x1, hidden width int(1.5 * C_in)) and the pointwise ``pw``."""

    def __init__(self, C_in: int, C_out: int, k_conv: Sequence[int]) -> None:
        super().__init__()
        self.conv_list = nn.ModuleList([nn.Conv2d(C_in, C_in, k, stride=1, padding=k // 2, groups=C_in) for k in k_conv])
        hid = int(1.5 * C_in)
        self.ffn1 = nn.Sequential(nn.Conv2d(C_in, hid, 1), nn.GELU(), nn.Conv2d(hid, C_in, 1))
        self.pw = nn.Conv2d(C_in, C_in, 1)
        self.ffn2 = nn.Sequential(nn.Conv2d(C_in, hid, 1), nn.GELU(), nn.Conv2d(hid, C_out, 1))

    forward = _no_forward


class SKMotionEncoder6_Deep_nopool_res(nn.Module):
    def __init__(self, corr_levels: int, corr_radius: int, k_conv: Sequence[int]) -> None:
        super().__init__()
        planes = corr_levels * (2 * corr_radius + 1) ** 2
        self.convc1 = PCBlock4_Deep_nopool_res(planes, 256, k_conv=k_conv)
        self.convc2 = PCBlock4_Deep_nopool_res(256, 192, k_conv=k_conv)
        self.convf1 = nn.Conv2d(2, 128, 1, 1, 0)
        self.convf2 = PCBlock4_Deep_nopool_res(128, 64, k_conv=k_conv)
        self.conv = PCBlock4_Deep_nopool_res(64 + 192, 128 - 2, k_conv=k_conv)

    forward = _no_forward


class SKUpdateBlock6_Deep_nopoolres_AllDecoder(nn.Module):
    def __init__(self, corr_levels: int, corr_radius: int, k_conv: Sequence[int], PCUpdater_conv: Sequence[int], num_heads: int,
                 hidden_dim: int = 128) -> None:
        super().__init__()
        self.encoder = SKMotionEncoder6_Deep_nopool_res(corr_levels, corr_radius, k_conv)
        self.gru = PCBlock4_Deep_nopool_res(128 + hidden_dim + hidden_dim + 128, 128, k_conv=PCUpdater_conv)
        self.flow_head = PCBlock4_Deep_nopool_res(128, 2, k_conv=k_conv)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1, padding=0))
        self.aggregator = Aggregate(dim=128, dim_head=128, heads=num_heads)

    forward = _no_forward


def _check_kernels(name: str, ks: Sequence[int]) -> tuple:
    ks = tuple(ks)
    bad = [k for k in ks if not isinstance(k, int) or isinstance(k, bool) or k < 1 or k > 31 or k % 2 == 0]
    if bad or len(ks) > 8:
        raise ValueError(f"skflow: {name} entries must be odd kernel sizes in 1..31 (at most 8 of them); got {ks}")
    return ks


class SKFlow(GMA):
    pretrained_checkpoints = {
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/skflow-kitti-4e1f8b63.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/skflow-sintel-98fb67cf.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/skflow-things-f84e6538.ckpt",
    }
    _variant = _lib.VARIANT_SKFLOW
    _engine_cls = SKFlowEngine

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, k_conv: Sequence[int] = (1, 15), PCUpdater_conv: Sequence[int] = (1, 7), num_heads: int = 1,
                 position_only: bool = False, position_and_content: bool = False, alternate_corr: bool = False, **kwargs) -> None:
        self.k_conv = _check_kernels("k_conv", k_conv)
        self.PCUpdater_conv = _check_kernels("PCUpdater_conv", PCUpdater_conv)
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow,
                         iters=iters, num_heads=num_heads, position_only=position_only, position_and_content=position_and_content,
                         alternate_corr=alternate_corr, **kwargs)

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        self.fnet = BasicEncoder(output_dim=256, norm_fn="instance", dropout=self.dropout)
        self.cnet = BasicEncoder(output_dim=self.hidden_dim + self.context_dim, norm_fn="batch", dropout=self.dropout)
        self.update_block = SKUpdateBlock6_Deep_nopoolres_AllDecoder(self.corr_levels, self.corr_radius, self.k_conv, self.PCUpdater_conv,
                                                                      self.num_heads, hidden_dim=self.hidden_dim)
        self.att = Attention(dim=self.context_dim, position_only=self.position_only, position_and_content=self.position_and_content,
                             heads=self.num_heads, max_pos_size=self.max_pos_size, dim_head=self.context_dim)


@register_model
@trainable
class skflow(SKFlow):
    pass
