"""CCMR and CCMR+ (MS-RAFT+'s multi-scale refinement with XCiT global context) on libptlflow_b200.

Surface kept from ptlflow/models/ccmr/ccmr.py:41-275: classes ``ccmr`` (3 scales, ``iters=[8, 10, 15]``) and ``ccmr_p`` (4 scales,
``iters=[8, 10, 10, 10]``), the constructor keywords (``corr_levels, corr_radius, iters, alternate_corr, lookup_pyramid_levels,
lookup_radius, model_type, cnet_norm, fnet_norm, num_scales``), the ``kitti`` / ``sintel`` checkpoint tables, the state_dict keys
(``fnet.*``, ``cnet.*``, ``update_block.*`` with ``update_block.aggregator.{i}``, and ``xcit.{i}``), ``forward(dict) -> dict`` with
``flows`` [B,1,2,H,W] and ``flow_small`` [B,2,int(H/16),int(W/16)], and the warm start from ``prev_preds.flow_small``.

Kernel mapping (DESIGN.md section 1, row a18): the encoders are ms_raft_p's (ccmr/extractor.py:62-274 adds a 1x1 conv with bias
after each up layer, and fnet's conv2 keeps 160 channels).  Per scale, one pfb_ccmr_refine call runs the context's XCiT, the
aggregator's folded attention, the iterations with the aggregator written into the GRU's motion_global columns, and the handover:
the convex 2x of the FLOW added to the finer grid (ccmr.py:195-202).  ``ccmr`` ends at 1/4 scale and adds one upflow2 (bilinear 2x,
align_corners=True).  Images are padded to multiples of 32 (output_stride = 32).
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn as nn

from ... import _lib
from ...engine import CCMREngine
from ...utils.registry import register_model, trainable
from ..ms_raft_plus.ms_raft_plus import MSRAFTPlus, _PyramidEncoder
from ..raft.update import BasicMotionEncoder, FlowHead, SepConvGRU, _no_forward

_SCALES = {"CCMR": 3, "CCMR+": 4}


class BasicEncoder_resconv(_PyramidEncoder):
    """fnet (ccmr/extractor.py:62-172): conv2 160 -> 160, up layers 128 / 96 / 64 each followed by a 1x1 of the same width."""

    def __init__(self, output_dim: int = 256, model_type: str = "CCMR+") -> None:
        super().__init__(output_dim, conv2_dim=160, after_up_dims=(128, 96, 64), num_up=_SCALES[model_type] - 1)


class Basic_Context_Encoder_resconv(_PyramidEncoder):
    """cnet (ccmr/extractor.py:175-274): conv2 160 -> output_dim, up layers 128 / 96 / 64 on ``output_dim + skip`` channels, each
    followed by a 1x1 to ``output_dim``."""

    def __init__(self, output_dim: int = 256, model_type: str = "CCMR+") -> None:
        super().__init__(output_dim, after_up_dims=(output_dim,) * 3, num_up=_SCALES[model_type] - 1)


class _PositionalEncodingFourier(nn.Module):
    def __init__(self, hidden_dim: int = 32, dim: int = 128) -> None:
        super().__init__()
        self.token_projection = nn.Conv2d(hidden_dim * 2, dim, kernel_size=1)

    forward = _no_forward


class _XCA(nn.Module):
    def __init__(self, dim: int, num_heads: int, separate: bool) -> None:
        super().__init__()
        self.temperature = nn.Parameter(torch.ones(num_heads, 1, 1))
        if separate:
            self.to_qk = nn.Linear(dim, 2 * dim)
            self.to_v = nn.Linear(dim, dim)
        else:
            self.qkv = nn.Linear(dim, 3 * dim)
        self.proj = nn.Linear(dim, dim)

    forward = _no_forward


class _Mlp(nn.Module):
    def __init__(self, dim: int) -> None:
        super().__init__()
        self.fc1 = nn.Linear(dim, dim)
        self.fc2 = nn.Linear(dim, dim)

    forward = _no_forward


class _LPI(nn.Module):
    def __init__(self, dim: int) -> None:
        super().__init__()
        self.conv1 = nn.Conv2d(dim, dim, 3, padding=1, groups=dim)
        self.bn = nn.GroupNorm(8, dim)
        self.conv2 = nn.Conv2d(dim, dim, 3, padding=1, groups=dim)

    forward = _no_forward


class _XCABlock(nn.Module):
    """XCABlock (xcit.py:242-300), eta = 1: LayerNorm eps 1e-6, 8 heads, mlp_ratio 1."""

    def __init__(self, dim: int, num_heads: int, separate: bool) -> None:
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = _XCA(dim, num_heads, separate)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = _Mlp(dim)
        self.norm3 = nn.LayerNorm(dim, eps=1e-6)
        self.local_mp = _LPI(dim)
        self.gamma1 = nn.Parameter(torch.ones(dim))
        self.gamma2 = nn.Parameter(torch.ones(dim))
        self.gamma3 = nn.Parameter(torch.ones(dim))

    forward = _no_forward


class XCiT(nn.Module):
    """XCiT(embed_dim=128, depth=1, num_heads=8, mlp_ratio=1) of xcit.py:304-427; ``separate`` is the aggregator's cross form."""

    def __init__(self, embed_dim: int = 128, num_heads: int = 8, separate: bool = False) -> None:
        super().__init__()
        self.blocks = nn.ModuleList([_XCABlock(embed_dim, num_heads, separate)])
        self.pos_embeder = _PositionalEncodingFourier(dim=embed_dim)

    forward = _no_forward


class BasicUpdateBlock(nn.Module):
    """ccmr/update.py:110-168: MS-RAFT+'s motion encoder, SepConvGRU(128, 384) on [inp | motion | motion_global], the flow head, the
    36-channel mask head and one aggregator XCiT per scale.  (RefineHead is defined there but never instantiated.)"""

    def __init__(self, levels: int, radius: int, hidden_dim: int = 128, num_scales: int = 4) -> None:
        super().__init__()
        self.encoder = BasicMotionEncoder(levels, radius)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=256 + 128)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 2 * 2 * 9, 1))
        self.aggregator = nn.ModuleList([XCiT(separate=True) for _ in range(num_scales)])

    forward = _no_forward


class CCMR(MSRAFTPlus):
    pretrained_checkpoints = {
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/ccmr-kitti-612444b9.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/ccmr-sintel-e1760f37.ckpt",
    }
    _variant = _lib.VARIANT_CCMR
    _engine_cls = CCMREngine
    _name = "ccmr"

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, iters: Sequence[int] = (8, 10, 15), alternate_corr: bool = True,
                 lookup_pyramid_levels: int = 2, lookup_radius: int = 4, model_type: str = "CCMR", cnet_norm: str = "group",
                 fnet_norm: str = "group", num_scales: int = 3, **kwargs) -> None:
        if cnet_norm != "group" or fnet_norm != "group":
            raise ValueError(f"{self._name}: cnet_norm / fnet_norm {cnet_norm!r} / {fnet_norm!r} are not supported; only the released "
                             f"'group' encoders are implemented (batch, instance and no normalisation are out of scope)")
        if model_type not in _SCALES or _SCALES[model_type] != num_scales:
            raise ValueError(f"{self._name}: model_type={model_type!r} with num_scales={num_scales} cannot run: the reference's 'CCMR' "
                             f"encoders give 3 scales and 'CCMR+' 4")
        self.num_scales, self.model_type, self.cnet_norm, self.fnet_norm = num_scales, model_type, cnet_norm, fnet_norm
        # the reference stores corr_levels / corr_radius as hyperparameters only; the lookups use lookup_pyramid_levels / radius
        self.ref_corr_levels, self.ref_corr_radius = corr_levels, corr_radius
        super().__init__(iters=iters, lookup_pyramid_levels=lookup_pyramid_levels, lookup_radius=lookup_radius, alternate_corr=alternate_corr,
                         **kwargs)
        self.output_stride = 32

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        self.fnet = BasicEncoder_resconv(output_dim=256, model_type=self.model_type)
        self.cnet = Basic_Context_Encoder_resconv(output_dim=256, model_type=self.model_type)
        self.update_block = BasicUpdateBlock(self.corr_levels, self.corr_radius, hidden_dim=128, num_scales=self.num_scales)
        self.xcit = nn.ModuleList([XCiT(separate=False) for _ in range(self.num_scales)])

    def _extra_engine_args(self):
        return {"xcit": self.xcit}

    def _loop_parameters(self):
        return list(self.update_block.parameters()) + list(self.xcit.parameters())


class CCMRPlus(CCMR):
    pretrained_checkpoints = {
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/ccmr+-kitti-c289d5e6.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/ccmr+-sintel-055b44ec.ckpt",
    }
    _name = "ccmr_p"

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, iters: Sequence[int] = (8, 10, 10, 10), alternate_corr: bool = True,
                 lookup_pyramid_levels: int = 2, lookup_radius: int = 4, model_type: str = "CCMR+", cnet_norm: str = "group",
                 fnet_norm: str = "group", num_scales: int = 4, **kwargs) -> None:
        super().__init__(corr_levels, corr_radius, iters, alternate_corr, lookup_pyramid_levels, lookup_radius, model_type, cnet_norm,
                         fnet_norm, num_scales, **kwargs)


@register_model
@trainable
class ccmr(CCMR):
    pass


@register_model
@trainable
class ccmr_p(CCMRPlus):
    pass
