"""GMA (global motion aggregation) on libptlflow_b200 -- BASELINE.json configs[2].

Surface kept from ptlflow/models/gma/gma.py:50-222: class name ``gma``, constructor keywords
(``corr_levels, corr_radius, dropout, gamma, max_flow, iters, num_heads, position_only,
position_and_content, alternate_corr``), state_dict keys (``fnet.*, cnet.*, update_block.*`` incl.
``update_block.aggregator.{to_v.weight,gamma}``, ``att.{to_qk.weight,pos_emb.*}``), ``forward(dict) -> dict``.

Kernel mapping of the extras (SURVEY.md section 8(a) row a13):
  * attention logits  scale * q . k   == level 0 of pfb_corr_volume_build(q, k) (same wgmma GEMM as the
    correlation volume: 1/sqrt(dim_head) is its built-in scale), then an in-place row softmax;
  * per iteration  motion + gamma * attn @ to_v(motion)  == a 1x1 convolution over the N attention columns
    with the sample's v as weights and an AXPY epilogue, inside pfb_raft_refine (variant 2).
Only the registered default (content attention, one head) is implemented; the positional variants raise.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn

from ... import ops
from ...utils.registry import register_model, trainable
from ..raft.raft import RAFT
from ..raft.update import BasicMotionEncoder, FlowHead, SepConvGRU, _no_forward


class RelPosEmb(nn.Module):
    """Parameter container (gma_utils.py:6-30); only used by the positional attention variants."""

    def __init__(self, max_pos_size: int, dim_head: int) -> None:
        super().__init__()
        self.rel_height = nn.Embedding(2 * max_pos_size - 1, dim_head)
        self.rel_width = nn.Embedding(2 * max_pos_size - 1, dim_head)
        idx = torch.arange(max_pos_size)
        self.register_buffer("rel_ind", idx.view(1, -1) - idx.view(-1, 1) + max_pos_size - 1)

    forward = _no_forward


class Attention(nn.Module):
    def __init__(self, *, dim: int, position_only: bool, position_and_content: bool, max_pos_size: int = 100,
                 heads: int = 4, dim_head: int = 128) -> None:
        super().__init__()
        self.position_only, self.position_and_content = position_only, position_and_content
        self.heads, self.dim_head = heads, dim_head
        self.scale = dim_head ** -0.5
        self.to_qk = nn.Conv2d(dim, heads * dim_head * 2, 1, bias=False)
        self.pos_emb = RelPosEmb(max_pos_size, dim_head)

    forward = _no_forward


class Aggregate(nn.Module):
    def __init__(self, dim: int, heads: int = 4, dim_head: int = 128) -> None:
        super().__init__()
        self.heads = heads
        inner = heads * dim_head
        self.to_v = nn.Conv2d(dim, inner, 1, bias=False)
        self.gamma = nn.Parameter(torch.zeros(1))
        self.project = nn.Conv2d(inner, dim, 1, bias=False) if dim != inner else None

    forward = _no_forward


class GMAUpdateBlock(nn.Module):
    def __init__(self, corr_levels: int, corr_radius: int, num_heads: int, hidden_dim: int = 128) -> None:
        super().__init__()
        self.encoder = BasicMotionEncoder(corr_levels, corr_radius)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim + hidden_dim)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1))
        self.aggregator = Aggregate(dim=128, dim_head=128, heads=num_heads)

    forward = _no_forward


class GMA(RAFT):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/gma-chairs-d4ec321d.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/gma-things-90aafb63.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/gma-sintel-98d6f3d0.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/gma-kitti-8ca3ec80.ckpt",
    }
    _variant = 2

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8,
                 max_flow: float = 400, iters: int = 32, num_heads: int = 1, position_only: bool = False,
                 position_and_content: bool = False, alternate_corr: bool = False, **kwargs) -> None:
        self.num_heads, self.position_only, self.position_and_content = num_heads, position_only, position_and_content
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow,
                         iters=iters, alternate_corr=alternate_corr, **kwargs)
        self.has_trained_on_ptlflow = False

    def _build_networks(self) -> None:
        super()._build_networks()
        self.update_block = GMAUpdateBlock(self.corr_levels, self.corr_radius, num_heads=self.num_heads, hidden_dim=self.hidden_dim)
        self.att = Attention(dim=self.context_dim, position_only=self.position_only, position_and_content=self.position_and_content,
                             heads=self.num_heads, max_pos_size=160, dim_head=self.context_dim)

    def _attention(self, inp: torch.Tensor, eng) -> torch.Tensor:
        """softmax(scale * q k^T) as [B*N, N] (gma_utils.py:58-76): two 1x1 GEMMs, the all-pairs GEMM, a row softmax."""
        if self.num_heads != 1 or self.position_only or self.position_and_content:
            raise NotImplementedError("ptlflow_b200 gma: only the registered default (content attention, num_heads=1) is implemented")
        B, H, W, C = inp.shape
        q = torch.empty_like(inp)
        k = torch.empty_like(inp)
        ops.conv2d([inp], eng.att_q, q, impl=self.kernel_impl)
        ops.conv2d([inp], eng.att_k, k, impl=self.kernel_impl)
        sim = ops.corr_volume_build(q, k, 1, impl=self.kernel_impl)[0]  # [B*N, H, W] = <q, k> / sqrt(dim_head)
        return ops.softmax_rows(sim.view(B * H * W, H * W))

    def _extra_engine_args(self) -> Dict:
        return {"attention_module": self.att}


@register_model
@trainable
class gma(GMA):
    pass
