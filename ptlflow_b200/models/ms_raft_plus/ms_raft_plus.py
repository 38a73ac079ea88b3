"""MS-RAFT+ (four-scale RAFT refinement, group-norm U-Net encoders) on libptlflow_b200.

Surface kept from ptlflow/models/ms_raft_plus/ms_raft_plus.py:62-231: class name ``ms_raft_p``, constructor keywords (``gamma,
max_flow, iters, lookup_pyramid_levels, lookup_radius, alternate_corr``), state_dict keys (``fnet.*``, ``cnet.*`` with the reference's
module names, ``update_block.*``), ``forward(dict) -> dict`` with ``flows`` [B,1,2,H,W] and ``flow_small`` [B,2,int(H/16),int(W/16)],
and the warm start from ``prev_preds.flow_small``.

Kernel mapping (DESIGN.md section 1, row a17): the encoders' convolutions run in cuDNN (the first one on this library's wgmma kernel
in f16 / bf16), every GroupNorm + ReLU (+ residual join) is pfb_group_norm_act, and each up layer's ``cat[resize(coarser), skip]`` is
one pfb_upsample2x_concat.  The scale loop (1/16, 1/8, 1/4, 1/2) runs RAFT's update block through pfb_msraft_refine, one call per
scale: the lookups are on the fly on the tensor cores (or the volume pyramid with ``alternate_corr=False``), the mask head runs on
the last iteration of each scale only, and the handover between scales is the convex 2x upsample of the absolute coordinates.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import _lib, ops
from ...engine import MSRaftEngine
from ...utils.registry import register_model, trainable
from ..raft.extractor import _Encoder, _EncConv, _block, _run
from ..raft.raft import RAFT, _cudnn_flags
from ..raft.update import BasicUpdateBlock, _no_forward

_GROUP = 8  # channels per group: every GroupNorm here is GroupNorm(C // 8, C), conv1's GroupNorm(8, 64) included
_VOLUME_MAX = 2 ** 31  # elements of a level-0 correlation volume the volume kernels are run on (B * N^2)


class ResidualBlock(nn.Module):
    """Parameter container of ms_raft_plus/extractor.py:6-57 (group norm).  ``norm3`` is registered both as ``norm3.*`` and as
    ``downsample.1.*``.  A block that changes the channel count at stride 1 returns its branch without the residual."""

    def __init__(self, in_planes: int, planes: int, stride: int = 1) -> None:
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes, 3, padding=1, stride=stride)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1)
        self.relu = nn.ReLU(inplace=True)
        self.norm1 = nn.GroupNorm(planes // _GROUP, planes)
        self.norm2 = nn.GroupNorm(planes // _GROUP, planes)
        self.downsample = None
        if stride != 1:
            self.norm3 = nn.GroupNorm(planes // _GROUP, planes)
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=stride), self.norm3)

    forward = _no_forward


class _PyramidEncoder(_Encoder):
    """BasicEncoder / Basic_Context_Encoder of ms_raft_plus/extractor.py:123-323: conv1 7x7 / 2 -> GroupNorm(8, 64) -> ReLU, layer1..4
    (64, 96, 128, 160 channels at 1/2 .. 1/16), conv2 1x1 -> ``output_dim``, then up_layer2 / 1 / 0 on cat[2x resize(coarser), skip].
    forward_pm returns the four pixel-major outputs at 1/16, 1/8, 1/4 and 1/2.

    CCMR's encoders (ccmr/extractor.py:62-274) are the same with ``conv2_dim`` (conv2's width, default ``output_dim``), a 1x1
    ``after_up_layer{k}_conv`` with bias after each up layer (``after_up_dims``, its output widths) and ``num_up`` = 2 (no up_layer0,
    three outputs) or 3."""

    up_dims: Sequence[int] = (128, 96, 64)

    def __init__(self, output_dim: int = 256, conv2_dim: Optional[int] = None, after_up_dims: Optional[Sequence[int]] = None,
                 num_up: int = 3) -> None:
        nn.Module.__init__(self)
        self.norm_fn = "group"
        self.norm1 = nn.GroupNorm(8, 64)
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3)
        self.relu1 = nn.ReLU(inplace=True)
        self.in_planes = 64
        self.layer1 = self._make_layer(64, 1)
        self.layer2 = self._make_layer(96, 2)
        self.layer3 = self._make_layer(128, 2)
        self.layer4 = self._make_layer(160, 2)
        c2 = output_dim if conv2_dim is None else conv2_dim
        self.conv2 = nn.Conv2d(160, c2, 1)
        up = self._up_dims(output_dim)
        self.num_up = num_up
        prev = c2
        for k, skip in zip(range(2, 2 - num_up, -1), (128, 96, 64)):  # up_layer2, 1 (, 0)
            self.in_planes = prev + skip
            setattr(self, f"up_layer{k}", self._make_layer(up[2 - k], 1))
            prev = up[2 - k]
            if after_up_dims is not None:
                setattr(self, f"after_up_layer{k}_conv", nn.Conv2d(up[2 - k], after_up_dims[2 - k], 1))
                prev = after_up_dims[2 - k]
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.GroupNorm):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def _up_dims(self, output_dim: int) -> Sequence[int]:
        return self.up_dims

    def _make_layer(self, dim: int, stride: int) -> nn.Sequential:
        layers = (ResidualBlock(self.in_planes, dim, stride), ResidualBlock(dim, dim, 1))
        self.in_planes = dim
        return nn.Sequential(*layers)

    # ---- inference path: planned convolutions (_EncConv) and this library's resize kernel ----
    def _plan(self, dtype, device):
        """(first convolution, [layer1..4 blocks], conv2, [(up layer's blocks, its after-up convolution or None)]) as steps.  The
        3x3s stay on cuDNN: pfb_enc_conv3x3 has no group-norm epilogue."""
        def blocks(name):  # a block that changes the channel count at stride 1 returns its branch without the residual
            return [_block(blk.downsample, [(blk.conv1, blk.norm1), (blk.conv2, blk.norm2)], dtype, device,
                           join=blk.conv1.in_channels == blk.conv2.out_channels or blk.downsample is not None) for blk in getattr(self, name)]

        def linear(conv):  # conv2 and CCMR's after-up 1x1s: convolution + bias
            return _EncConv(conv, None, dtype, device, relu=False)

        ups = []
        for k in range(2, 2 - self.num_up, -1):
            after = getattr(self, f"after_up_layer{k}_conv", None)
            ups.append((blocks(f"up_layer{k}"), None if after is None else linear(after)))
        return (_EncConv(self.conv1, self.norm1, dtype, device, native="first_conv7x7s2"), [blocks(f"layer{k}") for k in range(1, 5)],
                linear(self.conv2), ups)

    def forward_pm(self, x: torch.Tensor):
        """x: pixel-major frames [N,H,W,Cf] (H, W multiples of 16; channels past RGB zero) -> [1/16, 1/8, 1/4, 1/2] features."""
        first, down, conv2, ups = self._prepared(x.dtype, x.device)
        skips = [first(x)]
        for blocks in down:
            skips.append(_run(blocks, skips[-1]))
        outs = [conv2(skips.pop())]
        for blocks, after in ups:  # each on cat[2x resize(coarser), skip]: e3, e2, e1
            u = _run(blocks, ops.upsample2x_concat(outs[-1], skips.pop()))
            outs.append(u if after is None else after(u))
        return outs

    forward = _no_forward


class BasicEncoder(_PyramidEncoder):
    """fnet: 256, 128, 96 and 64 channels at 1/16 .. 1/2."""


class Basic_Context_Encoder(_PyramidEncoder):
    """cnet: ``output_dim`` channels at every scale."""

    def _up_dims(self, output_dim: int) -> Sequence[int]:
        return (output_dim,) * 3


class MSRAFTPlus(RAFT):
    pretrained_checkpoints = {
        "mixed": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/ms_raft_plus-mixed-2bb01f62.ckpt"
    }
    _variant = _lib.VARIANT_MS_RAFT_P
    _engine_cls = MSRaftEngine
    _name = "ms_raft_p"
    num_scales = 4  # 1/16, 1/8, 1/4, 1/2

    def __init__(self, gamma: float = 0.8, max_flow: float = 400, iters: Sequence[int] = (4, 6, 5, 10), lookup_pyramid_levels: int = 2,
                 lookup_radius: int = 4, alternate_corr: bool = True, **kwargs) -> None:
        _check_iters(iters, self.num_scales, self._name)
        super().__init__(corr_levels=lookup_pyramid_levels, corr_radius=lookup_radius, gamma=gamma, max_flow=max_flow, iters=iters,
                         alternate_corr=alternate_corr, **kwargs)
        self.output_stride = 16
        self.has_trained_on_ptlflow = False
        self.correlation_depth = lookup_pyramid_levels * (2 * lookup_radius + 1) ** 2

    # a list (a JSON config, a CLI parser) is kept as a tuple: the CUDA-graph cache keys on it
    @property
    def iters(self):
        return self._iters

    @iters.setter
    def iters(self, v) -> None:
        self._iters = tuple(v) if isinstance(v, (list, tuple)) else v

    # the reference's names for RAFT's corr_levels / corr_radius
    @property
    def lookup_pyramid_levels(self) -> int:
        return self.corr_levels

    @lookup_pyramid_levels.setter
    def lookup_pyramid_levels(self, v: int) -> None:
        self.corr_levels = v

    @property
    def lookup_radius(self) -> int:
        return self.corr_radius

    @lookup_radius.setter
    def lookup_radius(self, v: int) -> None:
        self.corr_radius = v

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        self.fnet = BasicEncoder(output_dim=256)
        self.cnet = Basic_Context_Encoder(output_dim=256)
        self.update_block = BasicUpdateBlock(self.corr_levels, self.corr_radius, hidden_dim=128)
        self.update_block.mask[2] = nn.Conv2d(256, 2 * 2 * 9, 1)  # scale = 2 (ms_raft_plus/update.py:144-148)

    def _grid16(self, h: int, w: int):
        """The padded 1/16-resolution grid of h x w images (images are padded to multiples of output_stride)."""
        s = self.output_stride
        return -(-h // s) * (s // 16), -(-w // s) * (s // 16)

    def _check_grid(self, h: int, w: int) -> None:
        """h, w: the grid at output_stride, after padding."""
        _check_iters(self.iters, self.num_scales, self._name)
        n = 2 ** (self.corr_levels - 1)
        f = self.output_stride // 16
        h16, w16 = f * h, f * w
        if h16 < n or w16 < n:
            raise ValueError(f"{self._name}: the 1/16-resolution grid {h16}x{w16} is smaller than 2**(lookup_pyramid_levels - 1) = {n} "
                             f"on a side; pad the images to at least {16 * n} px per side")

    def forward(self, inputs):
        images = inputs["images"]
        prev = inputs.get("prev_preds")
        if prev is not None and prev.get("flow_small") is not None:
            h, w = images.shape[-2:]
            grid = self._grid16(h, w)
            fs = tuple(prev["flow_small"].shape[-2:])
            if fs != grid:
                # the reference adds the warm start on the padded 1/16 grid, so it fails unless H and W are multiples of the padding
                raise ValueError(f"{self._name}: the warm start flow_small is {fs[0]}x{fs[1]} but the padded 1/16 grid of {h}x{w} images "
                                 f"is {grid[0]}x{grid[1]}; warm starts need H and W that are multiples of {self.output_stride}")
        return super().forward(inputs)

    def _forward_device_impl(self, images: torch.Tensor, flow_init: Optional[torch.Tensor], scratch: Optional[dict]):
        """images [B,2,3,H,W] on the device -> (flow_up fp32 [B,2,H,W], flow_small fp32 [B,2,H//16,W//16]); enqueued without host
        synchronisation, so the whole forward is one CUDA graph (ms_raft_plus.py:146-226, ccmr.py:141-230 in eval)."""
        from ...utils.utils import InputPadder

        resizer = InputPadder(images.shape, stride=self.output_stride, pad_mode="replicate", two_side_pad=True)
        B = images.shape[0]
        frames = ops.preprocess_frames(images, resizer.tgt_size, resizer.pad_top_left, out_channels=self.frame_channels)
        strict = frames.dtype == torch.float32 and self.strict_fp32
        with _cudnn_flags(self.cudnn_benchmark, not strict):
            fpyr = self.fnet.forward_pm(frames)  # both frames as one batch: GroupNorm is per sample
            cpyr = self.cnet.forward_pm(frames[:B])
        eng = self._get_engine(frames.dtype, frames.device)
        out_hw = tuple(images.shape[-2:])
        h16, w16 = fpyr[0].shape[1:3]
        coords = ops.init_coords(B, h16, w16, frames.device, flow_init)
        S = self.num_scales
        fine = 2 ** (S - 1)
        # one workspace, planned for the finest (largest) scale, serves the calls of every scale in turn
        ws = eng.workspace(eng.make_cfg(B, fine * h16, fine * w16, 1, out_hw, resizer.pad_top_left, self.alternate_corr, 128), scratch)
        for i in range(S):
            f = fpyr[i]
            C = f.shape[-1]
            fmap1, fmap2 = f[:B], f[B:]
            net, inp = ops.context_split(cpyr[i], self.hidden_dim, self.context_dim)
            if self.alternate_corr:
                if C % 64 and frames.dtype != torch.float32:
                    # 96 channels at 1/4 (and ccmr's 160 at 1/16): rows of a multiple of 64 with zero channels, so the tensor-core
                    # lookup serves the scale; the dot products are unchanged and the scale stays 1/sqrt(C)
                    fmap1, fmap2 = F.pad(fmap1, (0, 64 - C % 64)), F.pad(fmap2, (0, 64 - C % 64))
                pyramid, layout, f1 = ops.feature_pyramid(fmap2.contiguous(), self.corr_levels), 0, fmap1.contiguous()
            else:
                (pyramid, layout), f1 = eng.build_volume(fmap1.contiguous(), fmap2.contiguous(), impl=self.kernel_impl), None
            last = i == S - 1
            # the last scale's convex 2x upsample reaches 1/2**(4 - S): bilinear 2x steps take it to full resolution
            res = eng.refine_scale(i, pyramid, layout, net, inp, coords, int(self.iters[i]), out_hw, resizer.pad_top_left, ws, fmap1=f1,
                                   corr_scale=1.0 / math.sqrt(C), last=last, upflow2=4 - S if last else 0, fork_flow=self.fork_flow)
            if not last:
                coords = res
        return res

    def _check_volume(self, images: torch.Tensor) -> None:
        if self.alternate_corr:
            return
        h16, w16 = self._grid16(*images.shape[-2:])
        fine = 2 ** (self.num_scales - 1)  # the finest scale's grid over the 1/16 one
        n = h16 * fine * w16 * fine
        if images.shape[0] * n * n >= _VOLUME_MAX:
            raise ValueError(f"{self._name}: alternate_corr=False needs a {images.shape[0]} x {n} x {n} correlation volume at the finest "
                             f"scale, more than the volume kernels address ({_VOLUME_MAX} elements); use alternate_corr=True")

    def _forward_device(self, images: torch.Tensor, flow_init: Optional[torch.Tensor], scratch: Optional[dict] = None):
        self._check_volume(images)
        return super()._forward_device(images, flow_init, scratch)


def _check_iters(iters, num_scales: int, name: str) -> None:
    try:
        vals = [int(i) for i in iters]
    except TypeError:
        raise ValueError(f"{name}: iters must be a sequence of {num_scales} iteration counts, got {iters!r}") from None
    if len(vals) != num_scales or min(vals) < 1:
        raise ValueError(f"{name}: iters must hold num_scales = {num_scales} counts >= 1 (one per scale, coarsest first), got {tuple(iters)!r}")


@register_model
@trainable
class ms_raft_p(MSRAFTPlus):
    pass
