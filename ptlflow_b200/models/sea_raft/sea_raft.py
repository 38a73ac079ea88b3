"""SEA-RAFT (ConvNeXt refinement loop, ResNet-FPN encoders) on libptlflow_b200.

Surface kept from ptlflow/models/sea_raft/sea_raft.py:53-441: class names ``sea_raft``, ``sea_raft_s``, ``sea_raft_m``,
``sea_raft_l``, constructor keywords (``corr_levels, corr_radius, dim, initial_dim, num_blocks, block_dims, pretrain, gamma,
max_flow, iters, alternate_corr, use_var, var_min, var_max``), state_dict keys (``cnet.*, init_conv.*, upsample_weight.*,
flow_head.*`` and, when ``iters > 0``, ``fnet.*, update_block.{encoder, refine}.*``), ``forward(dict) -> dict`` with ``flows`` and
``flow_small``.  ``prev_preds`` is ignored, as in the reference: SEA-RAFT has no warm start.

Kernel mapping (DESIGN.md section 1, row a16): the encoders are ResNet-FPNs with every BatchNorm folded into its convolution
(cuDNN convolutions, this library's bias / ReLU / residual passes).  The correlation pyramid is RAFT's: SEA-RAFT halves fmap2
bilinearly before each level's volume (sea_raft/corr.py:77-83), which is a 2x2 mean, and the volume is linear in fmap2.
init_conv, the flow and mask heads, RAFT's motion encoder and every ConvNeXt block run in pfb_searaft_refine
(ptlflow_b200/engine.py SEARaftEngine); the depthwise convolution + LayerNorm is its own kernel.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn as nn

from ... import _lib, ops
from ...engine import SEARaftEngine
from ...utils.registry import register_model, trainable
from ..raft.extractor import _Encoder
from ..raft.raft import RAFT
from ..raft.update import BasicMotionEncoder, _no_forward

_BLOCKS = {"resnet18": (2, 2, 2), "resnet34": (3, 4, 6)}


class BasicBlock(nn.Module):
    """Parameter container of sea_raft/layer.py:126-150.  ``bn3`` is registered both as ``bn3.*`` and as ``downsample.1.*``."""

    def __init__(self, in_planes: int, planes: int, stride: int = 1) -> None:
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes, 3, stride=stride, padding=1)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1)
        self.bn1 = nn.BatchNorm2d(planes)
        self.bn2 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = None
        if stride != 1 or in_planes != planes:
            self.bn3 = nn.BatchNorm2d(planes)
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=stride), self.bn3)

    forward = _no_forward


class ResNetFPN(_Encoder):
    """sea_raft/extractor.py:6-116 with BatchNorm: conv1 7x7 / 2 -> bn1 -> ReLU -> three stages of BasicBlocks (1/2, 1/4, 1/8) ->
    final_conv 1x1.  Inference through _Encoder.forward_pm: every BatchNorm folded into its convolution (eval mode)."""

    enc_conv3x3 = False  # its stride-1 3x3 layers stay on cuDNN, the 64 -> 64 and 128 -> 128 ones pfb_enc_conv3x3 supports included

    def __init__(self, block_dims: Sequence[int], initial_dim: int, pretrain: str, input_dim: int = 3, output_dim: int = 256) -> None:
        nn.Module.__init__(self)
        self.norm_fn = "batch"
        dims = [int(d) for d in block_dims]  # (the reference scales the caller's list in place; this copy leaves it alone)
        self.conv1 = nn.Conv2d(input_dim, initial_dim, 7, stride=2, padding=3)
        self.bn1 = nn.BatchNorm2d(initial_dim)
        self.relu = nn.ReLU(inplace=True)
        n = _BLOCKS[pretrain]
        self.in_planes = initial_dim
        self.layer1 = self._make_layer(dims[0], 1, n[0])
        self.layer2 = self._make_layer(dims[1], 2, n[1])
        self.layer3 = self._make_layer(dims[2], 2, n[2])
        self.final_conv = nn.Conv2d(dims[2], output_dim, 1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                nn.init.zeros_(m.bias)

    def _make_layer(self, dim: int, stride: int, num: int) -> nn.Sequential:
        layers = [BasicBlock(self.in_planes, dim, stride)] + [BasicBlock(dim, dim, 1) for _ in range(num - 1)]
        self.in_planes = dim
        return nn.Sequential(*layers)

    def _layers(self):
        blocks = [(blk.downsample, [(blk.conv1, blk.bn1), (blk.conv2, blk.bn2)]) for blk in (*self.layer1, *self.layer2, *self.layer3)]
        return (self.conv1, self.bn1), blocks, self.final_conv

    forward = _no_forward


class LayerNorm(nn.Module):
    """Parameter container of sea_raft/layer.py:86-113 (channels_last)."""

    def __init__(self, normalized_shape: int, eps: float = 1e-6) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))
        self.eps = eps

    forward = _no_forward


class ConvNextBlock(nn.Module):
    """Parameter container of sea_raft/layer.py:41-83: dwconv 7x7 -> LayerNorm -> pwconv1 (Linear, 4 * output_dim) -> GELU ->
    pwconv2 (Linear) -> gamma -> final(x + .) (1x1)."""

    def __init__(self, dim: int, output_dim: int, layer_scale_init_value: float = 1e-6) -> None:
        super().__init__()
        self.dwconv = nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, 4 * output_dim)
        self.pwconv2 = nn.Linear(4 * output_dim, dim)
        self.gamma = nn.Parameter(layer_scale_init_value * torch.ones((dim)))
        self.final = nn.Conv2d(dim, output_dim, kernel_size=1, padding=0)

    forward = _no_forward


class SEAUpdateBlock(nn.Module):
    """Parameter container of sea_raft/update.py:39-54: RAFT's motion encoder and ``num_blocks`` ConvNextBlocks ``refine``."""

    def __init__(self, corr_levels: int, corr_radius: int, num_blocks: int, hdim: int = 128, cdim: int = 128) -> None:
        super().__init__()
        self.encoder = BasicMotionEncoder(corr_levels, corr_radius)  # RAFT's, at dim = 128
        self.refine = nn.ModuleList([ConvNextBlock(2 * cdim + hdim, hdim) for _ in range(num_blocks)])

    forward = _no_forward


class SEARAFT(RAFT):
    pretrained_checkpoints: dict = {}
    _variant = _lib.VARIANT_SEA_RAFT
    _engine_cls = SEARaftEngine

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dim: int = 128, initial_dim: int = 64, num_blocks: int = 2,
                 block_dims: Sequence[int] = (64, 128, 256), pretrain: str = "resnet18", gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 4, alternate_corr: bool = False, use_var: bool = True, var_min: float = 0, var_max: float = 10,
                 **kwargs) -> None:
        if dim != 128:
            raise ValueError(f"sea_raft: dim={dim} is not supported (the update block runs with dim = 128)")
        if pretrain not in _BLOCKS:
            raise ValueError(f"sea_raft: pretrain={pretrain!r} must be one of {sorted(_BLOCKS)}")
        if len(block_dims) != 3:
            raise ValueError(f"sea_raft: block_dims needs three entries, got {block_dims!r}")
        if not 1 <= num_blocks <= 8:
            raise ValueError(f"sea_raft: num_blocks={num_blocks} must be in 1..8")
        self.dim, self.initial_dim, self.num_blocks = dim, initial_dim, num_blocks
        self.block_dims, self.pretrain = block_dims, pretrain
        self.use_var, self.var_min, self.var_max = use_var, var_min, var_max
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, gamma=gamma, max_flow=max_flow, iters=iters,
                         alternate_corr=alternate_corr, **kwargs)

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = self.dim
        self.cnet = ResNetFPN(self.block_dims, self.initial_dim, self.pretrain, input_dim=6, output_dim=2 * self.dim)
        self.init_conv = nn.Conv2d(2 * self.dim, 2 * self.dim, 3, padding=1)
        self.upsample_weight = nn.Sequential(nn.Conv2d(self.dim, self.dim * 2, 3, padding=1), nn.ReLU(inplace=True),
                                             nn.Conv2d(self.dim * 2, 64 * 9, 1, padding=0))
        self.flow_head = nn.Sequential(nn.Conv2d(self.dim, 2 * self.dim, 3, padding=1), nn.ReLU(inplace=True),
                                       nn.Conv2d(2 * self.dim, 6, 3, padding=1))
        if self.iters > 0:
            self.fnet = ResNetFPN(self.block_dims, self.initial_dim, self.pretrain, input_dim=3, output_dim=2 * self.dim)
            self.update_block = SEAUpdateBlock(self.corr_levels, self.corr_radius, self.num_blocks, self.dim, self.dim)

    # -- engine: packs init_conv, the heads and (iters > 0) the update block --------------------
    def _loop_parameters(self):
        mods = [self.init_conv, self.flow_head, self.upsample_weight] + ([self.update_block] if hasattr(self, "update_block") else [])
        return [p for m in mods for p in m.parameters()]

    def _engine_module(self) -> nn.Module:
        return self

    def _check_grid(self, h8: int, w8: int) -> None:
        """The reference halves fmap2 corr_levels - 1 times and fails once a side reaches zero (e.g. an 8 x 12 grid at 64 x 96)."""
        n = 2 ** self.corr_levels
        if self.iters > 0 and (h8 < n or w8 < n):
            raise ValueError(f"sea_raft: the 1/8-resolution grid {h8}x{w8} is smaller than 2**corr_levels = {n} on a side; "
                             f"pad the images to at least {8 * n} px per side")

    def _forward_device_impl(self, images: torch.Tensor, flow_init: Optional[torch.Tensor], scratch: Optional[dict]):
        """images [B,2,3,H,W] on the device -> (flow_up fp32 [B,2,H,W], flow_small fp32 [B,2,H/8,W/8]); one CUDA graph per shape
        like RAFT's (sea_raft.py:165-276 in eval)."""
        from ...utils.utils import InputPadder

        resizer = InputPadder(images.shape, stride=self.output_stride, pad_mode="replicate", two_side_pad=True)
        B = images.shape[0]
        frames = ops.preprocess_frames(images, resizer.tgt_size, resizer.pad_top_left, out_channels=self.frame_channels)
        pair = torch.cat([frames[:B, ..., :3], frames[B:, ..., :3]], dim=-1)  # cnet sees cat[image1, image2] (sea_raft.py:190)
        # RAFT's encoder schedule (chunks, fnet beside cnet on a second stream, the fp32 context mode); fnet takes both frames as
        # one batch, which is exact because eval-mode BatchNorm is per channel
        fmap1, fmap2, cnet = self._encode(frames, B, cnet_in=pair, with_fnet=self.iters > 0)
        _, H8, W8, _ = cnet.shape
        eng = self._get_engine(cnet.dtype, cnet.device)
        coords = ops.init_coords(B, H8, W8, cnet.device)
        pyramid, layout, f1 = [], 0, None
        if self.iters > 0:
            if self.alternate_corr:
                pyramid, f1 = ops.feature_pyramid(fmap2, self.corr_levels), fmap1
            else:
                pyramid, layout = eng.build_volume(fmap1, fmap2, impl=self.kernel_impl)
        net = torch.empty((B, H8, W8, self.dim), dtype=cnet.dtype, device=cnet.device)
        orig_h, orig_w = images.shape[-2:]
        flow_up, flow_small = eng.refine(pyramid, layout, net, cnet, coords, self.iters, (orig_h, orig_w), resizer.pad_top_left, fmap1=f1,
                                         scratch=scratch)
        return self.postprocess_predictions(flow_up, resizer, is_flow=True), flow_small

    def forward(self, inputs):
        inputs = {k: v for k, v in inputs.items() if k != "prev_preds"}  # no warm start in SEA-RAFT
        return super().forward(inputs)


class SEARAFT_S(SEARAFT):
    pretrained_checkpoints = {
        "tartan": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_s-tartan-f7e26f21.ckpt",
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_s-chairs-6980249f.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_s-things-a15c1713.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_s-sintel-bb63371a.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_s-kitti-3a96c1cc.ckpt",
        "spring": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_s-spring-4d13c106.ckpt",
    }


_M_CHECKPOINTS = {
    "tartan": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_m-tartan-e684ed5f.ckpt",
    "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_m-chairs-1cb7b11e.ckpt",
    "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_m-things-ac45dd7f.ckpt",
    "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_m-sintel-f8bb7e3f.ckpt",
    "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_m-kitti-e51f7603.ckpt",
    "spring": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/sea_raft_m-spring-de7c13e2.ckpt",
}


class SEARAFT_M(SEARAFT):
    pretrained_checkpoints = dict(_M_CHECKPOINTS)

    def __init__(self, pretrain: str = "resnet34", iters: int = 4, **kwargs) -> None:
        super().__init__(pretrain=pretrain, iters=iters, **kwargs)


class SEARAFT_L(SEARAFT):
    pretrained_checkpoints = dict(_M_CHECKPOINTS)  # the reference's table for sea_raft_l names the sea_raft_m files

    def __init__(self, pretrain: str = "resnet34", iters: int = 12, **kwargs) -> None:
        super().__init__(pretrain=pretrain, iters=iters, **kwargs)


@register_model
@trainable
class sea_raft(SEARAFT):
    pass


@register_model
@trainable
class sea_raft_s(SEARAFT_S):
    pass


@register_model
@trainable
class sea_raft_m(SEARAFT_M):
    pass


@register_model
@trainable
class sea_raft_l(SEARAFT_L):
    pass
