"""LLA-Flow (local similarity attention and the shift-aggregated correlation volume) on libptlflow_b200.

Surface kept from ptlflow/models/llaflow/llaflow.py:50-262: class names ``llaflow`` and ``llaflow_raft``, the constructor keywords
(``corr_levels, corr_radius, dropout, gamma, max_flow, iters, alternate_corr, gma``), the checkpoint tables, the state_dict keys
(``fnet.*``, ``cnet.*`` as RAFT's BasicEncoder, ``ls1/ls2.to_qk.weight``, ``s_lsa.to_f1/to_f2.weight``, ``lsa.to_v.weight``, ``lsa.gamma``,
``gamma``, ``update_block.*`` as GMA's (``gma=True``, one head) or RAFT's, and ``att.to_qk.weight`` with ``gma=True``: the reference's
Attention has no position embedding), ``forward(dict) -> dict`` and the warm start from ``prev_preds.flow_small``.

As in the reference, the keyword ``gamma`` is the sequence loss's decay (kept in the hparams), while the attribute and state_dict key
``gamma`` is the volume's mixing parameter, initialised to 0.  ``alternate_corr`` is accepted and ignored: the reference warns and always
builds the volume, because its CorrBlock is the only one that adds gamma corr2.

Kernel mapping (DESIGN.md section 1, row a22): encoders, pre-processing, CUDA-graph capture and the loop are RAFT's / GMA's.
LLAFlowEngine builds the volume from (fmap1, fmap2, inp) before the loop: the stacked query / key 1x1 convolution of ls1 | ls2,
pfb_local_similar (both 5 x 5 attention tables), lsa.to_v and pfb_local_aggregate (fmap2'), to_f1 / to_f2, pfb_shift_pack (the GEMM
operands) and pfb_shift_volume_tiled (f16 / bf16: K = 6656 on wgmma into the tiled pyramid) or pfb_corr_volume_build_ex (the dense
pyramid, SIMT).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn

from ... import _lib
from ...engine import LLAFlowEngine
from ...utils.registry import register_model, trainable
from ..gma.gma import GMA, Aggregate
from ..raft.raft import RAFT
from ..raft.update import BasicMotionEncoder, BasicUpdateBlock, FlowHead, SepConvGRU, _no_forward


class LocalSimilar(nn.Module):
    """Parameter container of aggregate.py:97-129 (dim 128, one head, 5 x 5 window)."""

    def __init__(self, dim: int = 128) -> None:
        super().__init__()
        self.to_qk = nn.Conv2d(dim, dim * 2, 1, bias=False)

    forward = _no_forward


class ShiftLSA(nn.Module):
    """Parameter container of aggregate.py:157-187."""

    def __init__(self, dim: int = 256) -> None:
        super().__init__()
        self.to_f1 = nn.Conv2d(dim, dim, 1, bias=False)
        self.to_f2 = nn.Conv2d(dim, dim, 1, bias=False)

    forward = _no_forward


class LSA(nn.Module):
    """Parameter container of aggregate.py:190-216."""

    def __init__(self, dim: int = 256) -> None:
        super().__init__()
        self.to_v = nn.Conv2d(dim, dim, 1, bias=False)
        self.gamma = nn.Parameter(torch.zeros(1))

    forward = _no_forward


class Attention(nn.Module):
    """llaflow/gma.py:32-63: GMA's content-only attention, without a position embedding."""

    position_only = position_and_content = False

    def __init__(self, dim: int = 128, heads: int = 1, dim_head: int = 128) -> None:
        super().__init__()
        self.heads, self.scale = heads, dim_head ** -0.5
        self.to_qk = nn.Conv2d(dim, heads * dim_head * 2, 1, bias=False)

    forward = _no_forward


class GMAUpdateBlock(nn.Module):
    """llaflow/update.py:125-160 (one aggregator head)."""

    def __init__(self, corr_levels: int, corr_radius: int, hidden_dim: int = 128) -> None:
        super().__init__()
        self.encoder = BasicMotionEncoder(corr_levels, corr_radius)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim + hidden_dim)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1))
        self.aggregator = Aggregate(dim=128, dim_head=128, heads=1)

    forward = _no_forward


class LLAFlow(RAFT):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_gma-chairs-c4225e37.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_gma-things-1cfce7fe.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_gma-sintel-4ca6e4a9.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_gma-kitti-ac312150.ckpt",
    }
    _engine_cls = LLAFlowEngine
    # GMA's attention settings, for GMA._attention: content only, one head (llaflow.py:106)
    num_heads, position_only, position_and_content = 1, False, False

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, alternate_corr: bool = False, gma: bool = True, **kwargs) -> None:
        if corr_levels != 4:
            # CorrBlock is built with its default 4 levels whatever corr_levels says (llaflow.py:177), while convc1 is sized from it
            raise ValueError(f"llaflow's pyramid always has 4 levels (the reference fails with any other corr_levels), got {corr_levels}")
        if iters < 1:
            raise ValueError(f"llaflow needs at least one iteration (the convex upsample reads the last mask), got iters={iters}")
        self.gma = gma
        self._variant = _lib.VARIANT_GMA if gma else _lib.VARIANT_RAFT
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow, iters=iters,
                         alternate_corr=alternate_corr, **kwargs)
        self.gamma = nn.Parameter(torch.tensor([0.0]))  # the volume's gamma (llaflow.py:95); the loss decay stays in the hparams
        self.has_trained_on_ptlflow = False

    def _build_networks(self) -> None:
        super()._build_networks()
        self.ls1 = LocalSimilar(dim=128)
        self.ls2 = LocalSimilar(dim=128)
        self.s_lsa = ShiftLSA(dim=256)
        self.lsa = LSA(dim=256)
        if self.gma:
            self.update_block = GMAUpdateBlock(self.corr_levels, self.corr_radius, hidden_dim=self.hidden_dim)
            self.att = Attention(dim=self.context_dim, heads=1, dim_head=self.context_dim)
        else:
            self.update_block = BasicUpdateBlock(self.corr_levels, self.corr_radius, hidden_dim=self.hidden_dim)
            self.att = None

    def _local_modules(self):
        return (self.ls1, self.ls2, self.lsa, self.s_lsa, self.gamma)

    def _loop_parameters(self):
        ps = list(self.update_block.parameters()) + [p for m in self._local_modules()[:4] for p in m.parameters()] + [self.gamma]
        return ps + (list(self.att.parameters()) if self.att is not None else [])

    def _extra_engine_args(self) -> Dict:
        return {"attention_module": self.att, "local": self._local_modules()}

    def _attention(self, inp: torch.Tensor, eng):
        return GMA._attention(self, inp, eng) if self.att is not None else None

    def _correlation(self, fmap1: torch.Tensor, fmap2: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, eng):
        # always the volume, whatever alternate_corr says (llaflow.py:108-111, 177)
        pyramid, layout = eng.lla_volume(fmap1, fmap2, inp, impl=self.kernel_impl)
        return pyramid, layout, None

    def _check_grid(self, h8: int, w8: int) -> None:
        # bilinear_sampler normalises by (W_l - 1) and (H_l - 1) of every level (llaflow/utils.py): a coarsest level of one pixel
        # divides by zero in the reference
        n = 2 ** self.corr_levels
        if min(h8, w8) < n:
            raise ValueError(f"llaflow needs a 1/8-resolution grid of at least {n} pixels per side (images of more than "
                             f"{8 * (n - 1)} px after padding); got {h8} x {w8}")


class LLAFlowRAFT(LLAFlow):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_raft-chairs-a720c578.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_raft-things-b6cb5f0e.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_raft-sintel-69c82cea.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/llaflow_raft-kitti-b8b43046.ckpt",
    }

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, alternate_corr: bool = False, gma: bool = False, **kwargs) -> None:
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow, iters=iters,
                         alternate_corr=alternate_corr, gma=gma, **kwargs)


@register_model
@trainable
class llaflow(LLAFlow):
    pass


@register_model
@trainable
class llaflow_raft(LLAFlowRAFT):
    pass
