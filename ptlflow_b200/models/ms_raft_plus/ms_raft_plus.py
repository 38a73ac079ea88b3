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

from ... import ops
from ...engine import MSRaftEngine
from ...utils.registry import register_model, trainable
from ..raft.extractor import _NATIVE_CONV1, _Encoder, _conv_pm
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

    # ---- inference path: cuDNN convolutions + this library's group norm / resize kernels ----
    def _prepare_locked(self, sig, dtype, device):
        f32 = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()  # noqa: E731

        def conv(c: nn.Conv2d, norm: Optional[nn.GroupNorm]):
            e = {"w": c.weight.detach().to(device=device, dtype=dtype).contiguous(memory_format=torch.channels_last), "b": f32(c.bias),
                 "stride": c.stride[0], "padding": c.padding[0]}
            if norm is not None:
                e["gamma"], e["beta"], e["eps"] = f32(norm.weight), f32(norm.bias), float(norm.eps)
                e["group"] = c.out_channels // norm.num_groups
            return e

        prep = {"conv1": conv(self.conv1, self.norm1), "conv2": conv(self.conv2, None), "layers": {}, "after": {}}
        ups = [f"up_layer{k}" for k in range(2, 2 - self.num_up, -1)]
        for name in ups:
            after = getattr(self, f"after_{name}_conv", None)
            if after is not None:
                prep["after"][name] = conv(after, None)
        for name in ["layer1", "layer2", "layer3", "layer4"] + ups:
            blocks = []
            for blk in getattr(self, name):
                e = {"conv1": conv(blk.conv1, blk.norm1), "conv2": conv(blk.conv2, blk.norm2),
                     "residual": blk.conv1.in_channels == blk.conv2.out_channels or blk.downsample is not None}
                if blk.downsample is not None:
                    e["down"] = conv(blk.downsample[0], blk.downsample[1])
                blocks.append(e)
            prep["layers"][name] = blocks
        if _NATIVE_CONV1 and dtype in (torch.float16, torch.bfloat16) and tuple(self.conv1.weight.shape) == (64, 3, 7, 7):
            prep["conv1_native"] = ops.pack_first_conv(self.conv1.weight.detach().to(device).float(), dtype)
        torch.cuda.current_stream(device).synchronize()  # the casts / pack ran on this thread's stream: finish before others see them
        self._prep_cache = (sig, prep)
        return prep

    @staticmethod
    def _conv_gn(x: torch.Tensor, e: dict, relu: bool = True, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        # the convolution without its bias; the group norm folds the bias into its statistics (unlike instance norm, a bias that
        # differs between the channels of a group is not removed by the group mean)
        y = _conv_pm(x, (e["w"],), e["stride"], e["padding"])
        return ops.group_norm_act(y, e["gamma"], e["beta"], e["group"], bias=e["b"], relu=relu, residual=residual, eps=e["eps"], out=y)

    def _layer(self, x: torch.Tensor, blocks) -> torch.Tensor:
        for e in blocks:
            xs = x
            if "down" in e:
                xs = self._conv_gn(x, e["down"], relu=False)
            y = self._conv_gn(x, e["conv1"])
            x = self._conv_gn(y, e["conv2"], relu=True, residual=xs if e["residual"] else None)
        return x

    def forward_pm(self, x: torch.Tensor):
        """x: pixel-major frames [N,H,W,Cf] (H, W multiples of 16; channels past RGB zero) -> [1/16, 1/8, 1/4, 1/2] features."""
        prep = self._prepared(x.dtype, x.device)
        c1 = prep["conv1"]
        if "conv1_native" in prep and x.shape[-1] == 4 and x.is_contiguous():
            # wgmma first convolution: its epilogue accumulates the per-(image, channel) sums the group norm combines
            ws = ops.instance_norm_workspace((x.shape[0], 0, 0, 64), x.device)
            y = ops.first_conv7x7s2(x, prep["conv1_native"], None, relu=False, stats_ws=ws)
            x = ops.group_norm_act(y, c1["gamma"], c1["beta"], c1["group"], bias=c1["b"], relu=True, eps=c1["eps"], out=y, stats_ws=ws)
        else:
            if x.shape[-1] != c1["w"].shape[1]:  # zero frame channels beyond RGB: pad the filter to match
                key = ("conv1_pad", x.shape[-1])
                if key not in prep:
                    w = torch.zeros((64, x.shape[-1], 7, 7), dtype=c1["w"].dtype, device=c1["w"].device)
                    w[:, :3] = c1["w"]
                    prep[key] = dict(c1, w=w.contiguous(memory_format=torch.channels_last))
                c1 = prep[key]
            x = self._conv_gn(x, c1)
        L = prep["layers"]
        e1 = self._layer(x, L["layer1"])
        e2 = self._layer(e1, L["layer2"])
        e3 = self._layer(e2, L["layer3"])
        x = self._layer(e3, L["layer4"])
        y = _conv_pm(x, (prep["conv2"]["w"],), 1, 0)
        e4 = ops.bias_act(y, prep["conv2"]["b"], relu=False, out=y)
        outs = [e4]
        for k, skip in zip(range(2, 2 - self.num_up, -1), (e3, e2, e1)):
            name = f"up_layer{k}"
            u = self._layer(ops.upsample2x_concat(outs[-1], skip), L[name])
            a = prep["after"].get(name)
            if a is not None:  # CCMR's 1x1 after_up_layer conv with its bias
                y = _conv_pm(u, (a["w"],), 1, 0)
                u = ops.bias_act(y, a["b"], relu=False, out=y)
            outs.append(u)
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
    _variant = 5
    _engine_cls = MSRaftEngine

    def __init__(self, gamma: float = 0.8, max_flow: float = 400, iters: Sequence[int] = (4, 6, 5, 10), lookup_pyramid_levels: int = 2,
                 lookup_radius: int = 4, alternate_corr: bool = True, **kwargs) -> None:
        _check_iters(iters)
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

    def _check_grid(self, h16: int, w16: int) -> None:
        _check_iters(self.iters)
        n = 2 ** (self.corr_levels - 1)
        if h16 < n or w16 < n:
            raise ValueError(f"ms_raft_p: the 1/16-resolution grid {h16}x{w16} is smaller than 2**(lookup_pyramid_levels - 1) = {n} on "
                             f"a side; pad the images to at least {16 * n} px per side")

    def forward(self, inputs):
        images = inputs["images"]
        prev = inputs.get("prev_preds")
        if prev is not None and prev.get("flow_small") is not None:
            h, w = images.shape[-2:]
            grid = (-(-h // 16), -(-w // 16))
            fs = tuple(prev["flow_small"].shape[-2:])
            if fs != grid:
                # the reference adds the warm start on the padded 1/16 grid, so it fails unless H and W are multiples of 16
                raise ValueError(f"ms_raft_p: the warm start flow_small is {fs[0]}x{fs[1]} but the padded 1/16 grid of {h}x{w} images is "
                                 f"{grid[0]}x{grid[1]}; warm starts need H and W that are multiples of 16")
        return super().forward(inputs)

    def _forward_device_impl(self, images: torch.Tensor, flow_init: Optional[torch.Tensor], scratch: Optional[dict]):
        """images [B,2,3,H,W] on the device -> (flow_up fp32 [B,2,H,W], flow_small fp32 [B,2,H//16,W//16]); enqueued without host
        synchronisation, so the whole forward is one CUDA graph (ms_raft_plus.py:146-226 in eval)."""
        from ...utils.utils import InputPadder

        resizer = InputPadder(images.shape, stride=self.output_stride, pad_mode="replicate", two_side_pad=True)
        B = images.shape[0]
        frames = ops.preprocess_frames(images, resizer.tgt_size, resizer.pad_top_left, out_channels=self.frame_channels)
        strict = frames.dtype == torch.float32 and self.strict_fp32
        with _cudnn_flags(self.cudnn_benchmark, not strict):
            fpyr = self.fnet.forward_pm(frames)  # both frames as one batch: GroupNorm is per sample
            cpyr = self.cnet.forward_pm(frames[:B])
        eng = self._get_engine(frames.dtype, frames.device)
        orig_h, orig_w = images.shape[-2:]
        h16, w16 = fpyr[0].shape[1:3]
        coords = ops.init_coords(B, h16, w16, frames.device, flow_init)
        # one workspace, planned for the finest (largest) scale, serves the four calls in turn
        ws = eng.workspace(eng.make_cfg(B, 8 * h16, 8 * w16, 1, (orig_h, orig_w), resizer.pad_top_left, self.alternate_corr, 128), scratch)
        out = None
        for i in range(4):
            f = fpyr[i]
            C = f.shape[-1]
            fmap1, fmap2 = f[:B], f[B:]
            net, inp = ops.context_split(cpyr[i], self.hidden_dim, self.context_dim)
            scale, layout = 1.0 / math.sqrt(C), 0
            if self.alternate_corr:
                if C % 64 and frames.dtype != torch.float32:
                    # 96 channels at 1/4: rows of 128 with zero channels, so the tensor-core lookup serves the scale; the dot
                    # products are unchanged and the scale stays 1/sqrt(96)
                    fmap1, fmap2 = F.pad(fmap1, (0, 64 - C % 64)), F.pad(fmap2, (0, 64 - C % 64))
                pyramid, f1 = ops.feature_pyramid(fmap2.contiguous(), self.corr_levels), fmap1.contiguous()
            else:
                pyramid, f1 = eng.build_volume(fmap1, fmap2, impl=self.kernel_impl), None
                layout = eng.volume_layout
            res = eng.refine_scale(pyramid, net, inp, coords, int(self.iters[i]), (orig_h, orig_w), resizer.pad_top_left, ws, fmap1=f1,
                                   corr_scale=scale, volume_layout=layout, last=i == 3)
            if i < 3:
                coords = res
            else:
                out = res
        return out

    def _check_volume(self, images: torch.Tensor) -> None:
        if self.alternate_corr:
            return
        h, w = -(-images.shape[-2] // 16) * 8, -(-images.shape[-1] // 16) * 8  # the 1/2-scale grid after padding
        n = h * w
        if images.shape[0] * n * n >= _VOLUME_MAX:
            raise ValueError(f"ms_raft_p: alternate_corr=False needs a {images.shape[0]} x {n} x {n} correlation volume at 1/2 scale, more "
                             f"than the volume kernels address ({_VOLUME_MAX} elements); use alternate_corr=True")

    def _forward_device(self, images: torch.Tensor, flow_init: Optional[torch.Tensor], scratch: Optional[dict] = None):
        self._check_volume(images)
        return super()._forward_device(images, flow_init, scratch)


def _check_iters(iters) -> None:
    try:
        vals = [int(i) for i in iters]
    except TypeError:
        raise ValueError(f"ms_raft_p: iters must be a sequence of four iteration counts, got {iters!r}") from None
    if len(vals) != 4 or min(vals) < 1:
        raise ValueError(f"ms_raft_p: iters must hold four counts >= 1 (1/16, 1/8, 1/4, 1/2 scale), got {tuple(iters)!r}")


@register_model
@trainable
class ms_raft_p(MSRAFTPlus):
    pass
