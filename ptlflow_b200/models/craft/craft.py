"""CRAFT (cross-attentional flow transformer) on libptlflow_b200.

Surface kept from ptlflow/models/craft/craft.py:50-382: class name ``craft``, the constructor keywords, the checkpoint table, the
state_dict keys (``fnet.*``, ``cnet.*`` as RAFT's BasicEncoder; ``f2_trans.*``, ``att.*`` and, with ``craft=True``, ``corr_fn.*`` as
setrans.py's CrossAttFeatTrans / ExpandedFeatTrans / SlidingPosBiases2D; ``update_block.*`` as GMA's with the aggregator
``update_block.aggregator.{input_skip_coeff, first_linear.weight, feat_softaggr.feat2score.*}``), ``forward(dict) -> dict`` and the
warm start from ``prev_preds.flow_small``.  ``num_heads`` is accepted and ignored, as in the reference with ``use_setrans``.

Kernel mapping (DESIGN.md section 1, row a23): encoders, pre-processing, CUDA-graph capture and the loop are RAFT's / GMA's
(PFB_VARIANT_GMA, one head per intra-frame mode).  CRAFTEngine runs the three attention sites: q / k 1x1 convolutions per mode,
head-major per-mode scores on pfb_corr_volume_build_ex, the device-side clamp flag, then
  * f2 transformer and intra-frame attention: pfb_craft_window_softmax (clamp, window bias, mask radius, row softmax); the f2
    transformer's P_m @ V_m as GMA's per-sample-weight 1x1 GEMMs and pfb_craft_mode_aggregate (soft-aggregate, skip, LayerNorm);
  * inter-frame volume: in f16 / bf16 with a tiled (radius, levels) pair and modes of 64-channel multiples, pfb_craft_volume_tiled
    (wgmma; clamp flag, statistics and normalised tiled pyramid in three passes over the K = 256 GEMM); otherwise per-mode scores
    and pfb_craft_volume_norm (clamp, bias, mode mix, LayerNorm over each sample's N^2 values), then RAFT's dense avg-pool pyramid;
    with ``craft=False`` RAFT's plain volume of fmap1 and fmap2'.
The per-iteration aggregator is GMA's multi-head aggregate ending in pfb_craft_mode_aggregate (pfb_raft_buffers.agg_score).
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn

from ... import _lib, ops
from ...engine import CRAFTEngine
from ...utils.registry import register_model, trainable
from ..raft.raft import RAFT
from ..raft.update import BasicMotionEncoder, FlowHead, SepConvGRU, _no_forward

MAX_GRID = 200  # SlidingPosBiases2D's index tables cover grids up to 200 x 200 (setrans.py:743)
MODES = (1, 2, 4)


class SoftAggregate(nn.Module):
    """LearnedSoftAggregate (setrans.py:320-341): the parameters of its feat2score."""

    def __init__(self, num_feat: int) -> None:
        super().__init__()
        self.feat2score = nn.Linear(num_feat, 1)

    forward = _no_forward


class ExpandedFeatTrans(nn.Module):
    """setrans.py:346-471 without FFN, with the input skip (CRAFT's f2 transformer and motion aggregator)."""

    def __init__(self, in_dim: int, feat_dim: int, num_modes: int) -> None:
        super().__init__()
        self.num_modes = num_modes
        self.first_linear = nn.Linear(in_dim, feat_dim * num_modes, bias=False)
        self.feat_softaggr = SoftAggregate(feat_dim)
        self.input_skip_coeff = nn.Parameter(torch.ones(1))

    forward = _no_forward


class CrossAttFeatTrans(nn.Module):
    """setrans.py:474-653: query / key (shared in the inter-frame volume), attn_softaggr for scores or probabilities of several modes,
    out_trans for the f2 transformer."""

    def __init__(self, dim: int, num_modes: int, pos_code_weight: float, qk_bias: bool = False, tie_qk: bool = False,
                 out_attn_only: bool = True) -> None:
        super().__init__()
        self.num_modes, self.pos_code_weight = num_modes, pos_code_weight
        self.query = nn.Linear(dim, dim, bias=qk_bias)
        self.key = nn.Linear(dim, dim, bias=qk_bias)
        if tie_qk:  # tie_qk_scheme "shared" (setrans.py:548-551): one parameter under both names
            self.key.weight = self.query.weight
            if qk_bias:
                self.key.bias = self.query.bias
        if out_attn_only and num_modes > 1:
            self.attn_softaggr = SoftAggregate(1)
        if not out_attn_only:
            self.out_trans = ExpandedFeatTrans(dim, dim, num_modes)

    forward = _no_forward


class SlidingPosBiases2D(nn.Module):
    """setrans.py:742-813: the (2R+1)^2 learned biases (the index tables are not built: the kernels compute the window)."""

    def __init__(self, radius: int) -> None:
        super().__init__()
        self.R = radius
        self.biases = nn.Parameter(torch.zeros(2 * radius + 1, 2 * radius + 1))

    forward = _no_forward


class VisPosEncoder(nn.Module):
    def __init__(self, radius: int) -> None:
        super().__init__()
        self.pos_coder = SlidingPosBiases2D(radius)

    forward = _no_forward


class SelfAttVisPosTrans(nn.Module):
    """setrans.py:656-710 (and TransCorrBlock, corr.py:141-151, which holds the same two submodules)."""

    def __init__(self, dim: int, num_modes: int, pos_code_weight: float, radius: int, **kw) -> None:
        super().__init__()
        self.setrans = CrossAttFeatTrans(dim, num_modes, pos_code_weight, **kw)
        self.vispos_encoder = VisPosEncoder(radius)

    forward = _no_forward


class GMAUpdateBlock(nn.Module):
    """craft/update.py:131-196 with use_setrans: the aggregator is an ExpandedFeatTrans over the intra-frame modes."""

    def __init__(self, corr_levels: int, corr_radius: int, num_modes: int, hidden_dim: int = 128) -> None:
        super().__init__()
        self.encoder = BasicMotionEncoder(corr_levels, corr_radius)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim + hidden_dim)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1))
        self.aggregator = ExpandedFeatTrans(128, 128, num_modes)

    forward = _no_forward


class CRAFT(RAFT):
    pretrained_checkpoints = {
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/craft-things-5a41930c.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/craft-sintel-ff8e6563.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/craft-kitti-4d99b0c1.ckpt",
    }
    _variant = _lib.VARIANT_GMA
    _engine_cls = CRAFTEngine

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, f1trans: str = "none", f2trans: str = "full", f2_attn_mask_radius: int = -1, f2_num_modes: int = 4,
                 f2_pos_code_weight: float = 0.5, inter_num_modes: int = 4, inter_pos_code_type: str = "bias",
                 inter_pos_code_weight: float = 0.5, intra_pos_code_type: str = "bias", intra_pos_code_weight: float = 1.0,
                 intra_num_modes: int = 4, craft: bool = True, inter_qk_have_bias: bool = True, num_heads: int = 1,
                 pos_bias_radius: int = 7, use_setrans: bool = True, **kwargs) -> None:
        if f2trans == "none":
            raise ValueError("craft needs f2trans='full' (with f2trans='none' the reference never sets corr_multiplier)")
        if f1trans != "none":
            raise ValueError(f"craft supports f1trans='none' only (the two-way volume of f1trans={f1trans!r} is not implemented)")
        if not use_setrans:
            raise ValueError("craft needs use_setrans=True (without it the reference never sets intra_trans_config)")
        if inter_pos_code_type != "bias" or intra_pos_code_type != "bias":
            raise ValueError(f"craft supports the 'bias' position codes only, got inter {inter_pos_code_type!r} / intra {intra_pos_code_type!r}")
        if corr_levels != 4:
            raise ValueError(f"craft's pyramid always has 4 levels (TransCorrBlock and CorrBlock build 4), got corr_levels={corr_levels}")
        if iters < 1:
            raise ValueError(f"craft needs at least one iteration (the convex upsample reads the last mask), got iters={iters}")
        for name, m in (("f2_num_modes", f2_num_modes), ("inter_num_modes", inter_num_modes), ("intra_num_modes", intra_num_modes)):
            if m not in MODES:
                raise ValueError(f"craft: {name} must be one of {MODES}, got {m}")
        if not 0 <= pos_bias_radius <= 15:
            raise ValueError(f"craft: pos_bias_radius must be in 0..15, got {pos_bias_radius}")
        self.f1trans, self.f2trans, self.f2_attn_mask_radius = f1trans, f2trans, f2_attn_mask_radius
        self.f2_num_modes, self.f2_pos_code_weight = f2_num_modes, f2_pos_code_weight
        self.inter_num_modes, self.inter_pos_code_type, self.inter_pos_code_weight = inter_num_modes, inter_pos_code_type, inter_pos_code_weight
        self.intra_pos_code_type, self.intra_pos_code_weight, self.intra_num_modes = intra_pos_code_type, intra_pos_code_weight, intra_num_modes
        self.craft, self.inter_qk_have_bias, self.num_heads = craft, inter_qk_have_bias, num_heads
        self.pos_bias_radius, self.use_setrans = pos_bias_radius, use_setrans
        if corr_radius == -1:  # the default CRAFT lookup radius (craft.py:113-115)
            corr_radius = 4
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow, iters=iters,
                         **kwargs)
        self.has_trained_on_ptlflow = False

    def _build_networks(self) -> None:
        super()._build_networks()
        R = self.pos_bias_radius
        if self.craft:
            self.corr_fn = SelfAttVisPosTrans(256, self.inter_num_modes, self.inter_pos_code_weight, R, qk_bias=self.inter_qk_have_bias,
                                              tie_qk=True)
        else:
            self.corr_fn = None
        self.f2_trans = SelfAttVisPosTrans(256, self.f2_num_modes, self.f2_pos_code_weight, R, out_attn_only=False)
        self.att = SelfAttVisPosTrans(128, self.intra_num_modes, self.intra_pos_code_weight, R)
        self.update_block = GMAUpdateBlock(self.corr_levels, self.corr_radius, self.intra_num_modes, hidden_dim=self.hidden_dim)

    def _check_grid(self, h8: int, w8: int) -> None:
        if max(h8, w8) > MAX_GRID:
            raise ValueError(f"craft supports 1/8-resolution grids up to {MAX_GRID} x {MAX_GRID} (images up to {8 * MAX_GRID} px per side "
                             f"after padding), as the reference's position-bias tables; got {h8} x {w8}")

    def _loop_parameters(self):
        mods = [self.update_block, self.att, self.f2_trans] + ([self.corr_fn] if self.corr_fn is not None else [])
        return [p for m in mods for p in m.parameters()]

    def _extra_engine_args(self) -> Dict:
        return {"attention_module": self.att, "f2_trans": self.f2_trans, "corr_trans": self.corr_fn}

    def _attention(self, inp: torch.Tensor, eng):
        return eng.attention_probs(eng.att, ops.layernorm(inp, eps=1e-12), -1, self.kernel_impl)

    def _correlation(self, fmap1: torch.Tensor, fmap2: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, eng):
        fmap2t = eng.f2_transform(fmap2, self.f2_attn_mask_radius, self.kernel_impl)
        if self.craft:
            pyramid, layout = eng.craft_volume(fmap1, fmap2t, self.kernel_impl)
            return pyramid, layout, None
        pyramid, layout = eng.build_volume(fmap1, fmap2t, impl=self.kernel_impl)
        return pyramid, layout, None


@register_model
@trainable
class craft(CRAFT):
    pass
