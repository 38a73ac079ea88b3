"""GMA (global motion aggregation) on libptlflow_b200 -- BASELINE.json configs[2].

Surface kept from ptlflow/models/gma/gma.py:50-222: class name ``gma``, constructor keywords
(``corr_levels, corr_radius, dropout, gamma, max_flow, iters, num_heads, position_only,
position_and_content, alternate_corr``), state_dict keys (``fnet.*, cnet.*, update_block.*`` incl.
``update_block.aggregator.{to_v.weight,gamma,project.weight}``, ``att.{to_qk.weight,pos_emb.*}``), ``forward(dict) -> dict``.

Kernel mapping of the extras (SURVEY.md section 8(a) row a13), for content, position_only and position_and_content attention
and any num_heads; the attention is head-major [heads * B * N, N]:
  * content logits  scale * q_h . k_h  == level 0 of one pfb_corr_volume_build over heads * B samples of head-major q / k (same
    wgmma GEMM as the correlation volume: 1/sqrt(dim_head) is its built-in scale); content only: an in-place row softmax;
  * positional logits  scale * q_h . rel_height[u - x + P - 1] + scale * q_h . rel_width[v - y + P - 1]  == per-query tables from
    a 1x1 convolution of inp with the embedding folded into its weights, added to the content logits (if any) by
    pfb_attention_softmax_relpos, which also normalises the rows.  Grids above max_pos_size (160) per side raise ValueError;
  * per iteration  motion + gamma * project(attn_h @ to_v(motion)_h)  == one 1x1 convolution per head over the N attention
    columns with the sample's v as weights, then project with an AXPY epilogue (one head: no project, AXPY directly), inside
    pfb_raft_refine (variant 2).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn

from ... import _lib, ops
from ...utils.registry import register_model, trainable
from ..raft.raft import RAFT
from ..raft.update import BasicMotionEncoder, FlowHead, SepConvGRU, _no_forward


class RelPosEmb(nn.Module):
    """Parameter container (gma_utils.py:6-30) of the positional attention variants; RaftEngine folds it into packed weights."""

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
        self.max_pos_size = 160  # fixed in the reference model (gma.py:107)
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow,
                         iters=iters, alternate_corr=alternate_corr, **kwargs)
        self.has_trained_on_ptlflow = False

    def _build_networks(self) -> None:
        super()._build_networks()
        self.update_block = GMAUpdateBlock(self.corr_levels, self.corr_radius, num_heads=self.num_heads, hidden_dim=self.hidden_dim)
        self.att = Attention(dim=self.context_dim, position_only=self.position_only, position_and_content=self.position_and_content,
                             heads=self.num_heads, max_pos_size=self.max_pos_size, dim_head=self.context_dim)

    def _check_grid(self, h8: int, w8: int) -> None:
        # the relative-position tables cover offsets up to max_pos_size - 1 (gma_utils.py:12-16); content attention has no limit
        if (self.position_only or self.position_and_content) and max(h8, w8) > self.max_pos_size:
            raise ValueError(f"gma with positional attention supports 1/8-resolution grids up to {self.max_pos_size} x {self.max_pos_size} "
                             f"(images up to {8 * self.max_pos_size} px per side after padding); got {h8} x {w8}")

    def _attention(self, inp: torch.Tensor, eng) -> torch.Tensor:
        """softmax over the keys of the attention logits, head-major [heads*B*N, N] (gma_utils.py:54-76).
        Content logits scale * q_h . k_h: per-head 1x1 GEMMs into head-major q / k, then one all-pairs GEMM over heads*B samples.
        Positional logits scale * q_h . E[key - query + P - 1] (row and column tables): a 1x1 GEMM with the embedding folded into
        the weights writes the per-query tables, and the relative-position softmax adds them to the content logits (if any)."""
        B, H, W, C = inp.shape
        heads, N = self.num_heads, H * W
        position = self.position_only or self.position_and_content
        sim = None
        if not self.position_only:
            q = torch.empty((heads, B, H, W, C), dtype=inp.dtype, device=inp.device)
            k = torch.empty_like(q)
            for h in range(heads):
                ops.conv2d([inp], eng.att_q[h], q[h], impl=self.kernel_impl)
                ops.conv2d([inp], eng.att_k[h], k[h], impl=self.kernel_impl)
            # [heads*B*N, H, W] = <q, k> / sqrt(dim_head)
            sim = ops.corr_volume_build(q.view(heads * B, H, W, C), k.view(heads * B, H, W, C), 1, impl=self.kernel_impl)[0]
            sim = sim.view(heads * B * N, N)
            if not position:
                return ops.softmax_rows(sim)
        P = self.max_pos_size
        npos = 2 * P - 1
        tables = torch.empty((heads, B, H, W, eng.att_pos[0].Cout_pad), dtype=torch.float32, device=inp.device)
        for h in range(heads):
            ops.conv2d([inp], eng.att_pos[h], tables[h], epilogue=_lib.EPI_LINEAR_F32, scale=self.att.scale, impl=self.kernel_impl)
        tables = tables.view(heads * B * N, -1)
        out = sim if sim is not None else torch.empty((heads * B * N, N), dtype=inp.dtype, device=inp.device)
        return ops.attention_softmax_relpos(sim, tables[:, :npos], tables[:, npos:2 * npos], H, W, P, out=out)

    def _extra_engine_args(self) -> Dict:
        return {"attention_module": self.att}


@register_model
@trainable
class gma(GMA):
    pass
