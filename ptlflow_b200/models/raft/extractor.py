"""Feature / context encoders (SURVEY.md 8(a) row a14: not on the named hot path, kept as
cuDNN modules in channels_last; parameter names and shapes equal the reference's
ptlflow/models/raft/extractor.py:122-267 so checkpoints load strictly)."""
from __future__ import annotations

import os
import threading
from typing import List, NamedTuple, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import _lib, ops


def _norm(kind: str, channels: int, groups: int = 8) -> nn.Module:
    if kind == "batch":
        return nn.BatchNorm2d(channels)
    if kind == "instance":
        return nn.InstanceNorm2d(channels)
    if kind == "group":
        return nn.GroupNorm(num_groups=groups, num_channels=channels)
    if kind == "none":
        return nn.Identity()
    raise ValueError(f"unknown norm_fn {kind!r}")


class ResidualBlock(nn.Module):
    """3x3 -> 3x3 with identity (or strided 1x1) shortcut.  ``project``: a 1x1 convolution + norm shortcut at stride 1 too (SCV's
    encoders, scv/extractor.py:6-59)."""

    def __init__(self, in_planes: int, planes: int, norm_fn: str = "group", stride: int = 1, project: bool = False) -> None:
        super().__init__()
        self.conv1 = nn.Conv2d(in_planes, planes, 3, stride=stride, padding=1)
        self.conv2 = nn.Conv2d(planes, planes, 3, padding=1)
        self.relu = nn.ReLU(inplace=True)
        g = planes // 8
        self.norm1, self.norm2 = _norm(norm_fn, planes, g), _norm(norm_fn, planes, g)
        self.downsample = None
        if stride != 1 or project:
            self.norm3 = _norm(norm_fn, planes, g)
            # the norm is shared: state_dict carries it as both norm3.* and downsample.1.* (as upstream)
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=stride), self.norm3)

    def forward(self, x):
        y = self.relu(self.norm1(self.conv1(x)))
        y = self.relu(self.norm2(self.conv2(y)))
        if self.downsample is not None:
            x = self.downsample(x)
        return self.relu(x + y)


class BottleneckBlock(nn.Module):
    """1x1 -> 3x3 -> 1x1 bottleneck used by the small encoder."""

    def __init__(self, in_planes: int, planes: int, norm_fn: str = "group", stride: int = 1) -> None:
        super().__init__()
        q = planes // 4
        self.conv1 = nn.Conv2d(in_planes, q, 1)
        self.conv2 = nn.Conv2d(q, q, 3, stride=stride, padding=1)
        self.conv3 = nn.Conv2d(q, planes, 1)
        self.relu = nn.ReLU(inplace=True)
        g = planes // 8
        self.norm1, self.norm2, self.norm3 = _norm(norm_fn, q, g), _norm(norm_fn, q, g), _norm(norm_fn, planes, g)
        self.downsample = None
        if stride != 1:
            self.norm4 = _norm(norm_fn, planes, g)
            self.downsample = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=stride), self.norm4)

    def forward(self, x):
        y = self.relu(self.norm1(self.conv1(x)))
        y = self.relu(self.norm2(self.conv2(y)))
        y = self.relu(self.norm3(self.conv3(y)))
        if self.downsample is not None:
            x = self.downsample(x)
        return self.relu(x + y)


_NATIVE_CONV1 = bool(int(os.environ.get("PFB_NATIVE_CONV1", "1")))
_NATIVE_CONV2 = bool(int(os.environ.get("PFB_NATIVE_CONV2", "1")))
# the residual blocks' 3x3 stride-1 convolutions on pfb_enc_conv3x3 (read at every call: tools/time_encoder_convs.py
# switches it to compare both paths in one process)
_NATIVE_ENC_CONV = bool(int(os.environ.get("PFB_NATIVE_ENC_CONV", "1")))
# (Cin, Cout) of eligible layers that stay on cuDNN unless the kernel also takes their residual join: at 96 output channels
# the kernel computes 128 MMA rows, and cuDNN measured faster on the plain convolution (DESIGN.md section 5)
_ENC_CONV_CUDNN_UNFUSED = frozenset({(96, 96)})
# batch-norm-folded convolutions without a residual join: cuDNN's own conv + bias + ReLU epilogue instead of a separate pass
_CUDNN_FUSED_RELU = bool(int(os.environ.get("PFB_CUDNN_FUSED_RELU", "1")))
_prep_lock = threading.Lock()


def _norm_kind(norm: Optional[nn.Module]) -> str:
    if isinstance(norm, nn.InstanceNorm2d):
        return "instance"
    if isinstance(norm, nn.GroupNorm):
        return "group"
    return "batch" if isinstance(norm, nn.BatchNorm2d) else "none"


def enc_conv_eligible(conv: nn.Conv2d, dtype: torch.dtype, fused_residual: bool = False) -> bool:
    """A 3x3 stride-1 "same" convolution that pfb_enc_conv3x3 runs in this storage type (f16 / bf16; Cin a multiple of 32,
    Cout 64, 96 or 128), and that cuDNN did not measure faster on.  ``fused_residual``: the layer's bias, ReLU and residual
    join would go into the kernel's epilogue (a batch-norm-folded block's second convolution)."""
    return (tuple(conv.kernel_size) == (3, 3) and tuple(conv.stride) == (1, 1) and tuple(conv.padding) == (1, 1)
            and tuple(conv.dilation) == (1, 1) and conv.groups == 1 and conv.padding_mode == "zeros"
            and (fused_residual or (conv.in_channels, conv.out_channels) not in _ENC_CONV_CUDNN_UNFUSED)
            and ops.enc_conv3x3_supported(conv.in_channels, conv.out_channels, dtype))


def route_conv(conv: nn.Conv2d, norm: str, relu: bool, residual: bool, dtype: torch.dtype, native: Optional[str] = None) -> str:
    """The kernel that runs an encoder convolution followed by ``norm`` ('instance', 'group', 'batch' (folded) or 'none'), ReLU
    and the residual join, in this storage type.  ``native``: the library kernel the encoder offers the layer ('first_conv7x7s2'
    for the 7x7 stride-2 first convolution, 'enc_conv3x3' for a residual block's convolutions, 'conv2d' for the 1x1 output
    projection, None for cuDNN only); it is taken where the layer is that kernel's.  Else the cuDNN route:
    'cudnn_convolution_relu' (cuDNN's bias + ReLU epilogue), or a cuDNN convolution and the norm pass 'instance_norm_act',
    'group_norm_act' or 'bias_act'."""
    half = dtype in (torch.float16, torch.bfloat16)
    geometry = (tuple(conv.kernel_size), tuple(conv.stride), tuple(conv.padding), tuple(conv.dilation), conv.groups)
    if native == "first_conv7x7s2" and _NATIVE_CONV1 and half and tuple(conv.weight.shape) == (64, 3, 7, 7) \
            and geometry == ((7, 7), (2, 2), (3, 3), (1, 1), 1):
        return native
    # its epilogues: none (the instance norm follows), bias + ReLU (+ the residual join)
    if (native == "enc_conv3x3" and relu and norm != "group"
            and enc_conv_eligible(conv, dtype, fused_residual=residual and norm != "instance")):
        return native
    # cuDNN picked an sm_80 kernel without shared-memory staging for the projection (50 us per encoder, ncu launch list r02f),
    # and its bias needed a pass of its own
    if (native == "conv2d" and _NATIVE_CONV2 and half and geometry[:3] == ((1, 1), (1, 1), (0, 0)) and norm == "none"
            and not relu and not residual and conv.in_channels % 64 == 0 and conv.out_channels % 32 == 0 and conv.out_channels <= 1024):
        return native
    if norm in ("instance", "group"):
        return norm + "_norm_act"
    if _CUDNN_FUSED_RELU and relu and not residual and half:
        return "cudnn_convolution_relu"
    return "bias_act"


def _conv_pm(x: torch.Tensor, weight: torch.Tensor, stride, padding) -> torch.Tensor:
    """cuDNN convolution on a pixel-major tensor [N,H,W,C] -> [N,H',W',C'] (channels_last in and out, no copies)."""
    y = F.conv2d(x.permute(0, 3, 1, 2), weight, None, stride=stride, padding=padding)
    y = y.permute(0, 2, 3, 1)
    return y if y.is_contiguous() else y.contiguous()


class _EncConv:
    """One encoder convolution with the norm, ReLU and residual join that follow it, planned once per storage type and device:
    ``route`` names the kernel (route_conv), ``cudnn_route`` the cuDNN route that runs where the input does not suit it.

    Operands: ``weight``, the filter in the storage type (channels_last) with an eval-mode batch norm folded in (y = s * conv(x)
    + t -> weight * s, bias * s + t); ``bias`` fp32, added by this library's kernels (or ignored in front of an instance norm,
    whose mean removes it); ``bias_storage``, its storage-type copy for cuDNN's fused epilogue; the group norm's affine;
    ``packed``, the library kernel's weights.  ``conv`` is the module it was planned from."""

    def __init__(self, conv: nn.Conv2d, norm: Optional[nn.Module], dtype: torch.dtype, device, relu: bool = True,
                 residual: bool = False, native: Optional[str] = None) -> None:
        self.conv, self.relu, self.residual = conv, relu, residual
        self.norm = _norm_kind(norm)
        self.route = route_conv(conv, self.norm, relu, residual, dtype, native)
        self.cudnn_route = route_conv(conv, self.norm, relu, residual, dtype)
        self.stride, self.padding = tuple(conv.stride), tuple(conv.padding)
        w = conv.weight.detach().to(device=device, dtype=torch.float32)
        b = conv.bias.detach().to(device=device, dtype=torch.float32) if conv.bias is not None else torch.zeros(w.shape[0], device=device)
        if self.norm == "batch":
            s = norm.weight.detach().float().to(device) / torch.sqrt(norm.running_var.detach().float().to(device) + norm.eps)
            t = norm.bias.detach().float().to(device) - norm.running_mean.detach().float().to(device) * s
            w = w * s.view(-1, 1, 1, 1)
            b = b * s + t
        self.weight = w.to(dtype).contiguous(memory_format=torch.channels_last)
        self.bias = b.contiguous()
        # cast once, not per call
        self.bias_storage = self.bias.to(dtype) if self.cudnn_route == "cudnn_convolution_relu" else None
        if self.norm == "group":
            self.gamma = norm.weight.detach().to(device=device, dtype=torch.float32).contiguous()
            self.beta = norm.bias.detach().to(device=device, dtype=torch.float32).contiguous()
            self.group, self.eps = conv.out_channels // norm.num_groups, float(norm.eps)
        if self.route == "first_conv7x7s2":
            self.packed = ops.pack_first_conv(w, dtype)
        elif self.route == "enc_conv3x3":  # from the fp32 fold, rounded to the storage type once, as the cuDNN filter
            self.packed = ops.PackedConv([ops.ConvWeights(w)], dtype, device, src_channels=[conv.in_channels])
        elif self.route == "conv2d":  # the bias goes into the kernel's epilogue
            self.packed = ops.PackedConv([conv], dtype, device, src_channels=[conv.in_channels])
        self._padded = {}  # frame channel count -> the filter zero-padded to it

    def __call__(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x [N,H,W,Cin] pixel-major -> [N,H',W',Cout]; ``residual`` (when the step takes the join) [N,H',W',Cout]."""
        if self.route == "first_conv7x7s2" and x.shape[-1] == 4 and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0 and x.is_contiguous():
            if self.norm in ("instance", "group"):  # the norm's per-(image, channel) sums come out of the kernel's epilogue
                ws = ops.instance_norm_workspace((x.shape[0], 0, 0, 64), x.device)
                y = ops.first_conv7x7s2(x, self.packed, None, relu=False, stats_ws=ws)
                return self._norm_act(y, stats_ws=ws)
            return ops.first_conv7x7s2(x, self.packed, self.bias, relu=self.relu)
        if (self.route == "enc_conv3x3" and _NATIVE_ENC_CONV and x.is_contiguous()
                and (residual is None or residual.is_contiguous())):
            if self.norm == "instance":
                return self._norm_act(ops.enc_conv3x3(x, self.packed), residual)
            epi = _lib.ENC_CONV_BIAS_RELU if residual is None else _lib.ENC_CONV_BIAS_RELU_RESIDUAL
            return ops.enc_conv3x3(x, self.packed, epi, bias=self.bias, residual=residual)
        if self.route == "conv2d" and x.is_contiguous():
            out = torch.empty(x.shape[:3] + (self.packed.Cout,), dtype=x.dtype, device=x.device)
            return ops.conv2d([x], self.packed, out, epilogue=_lib.EPI_LINEAR)
        w = self.weight
        if x.shape[-1] != w.shape[1]:  # frames carry zero channels beyond RGB (8-byte pixels): pad the filter to match
            if x.shape[-1] not in self._padded:
                wp = torch.zeros((w.shape[0], x.shape[-1]) + tuple(w.shape[2:]), dtype=w.dtype, device=w.device)
                wp[:, : w.shape[1]] = w
                self._padded[x.shape[-1]] = wp.contiguous(memory_format=torch.channels_last)
            w = self._padded[x.shape[-1]]
        if self.cudnn_route == "cudnn_convolution_relu":
            y = torch.cudnn_convolution_relu(x.permute(0, 3, 1, 2), w, self.bias_storage, self.stride, self.padding, (1, 1), 1)
            y = y.permute(0, 2, 3, 1)
            return y if y.is_contiguous() else y.contiguous()
        # no bias in the convolution: PyTorch would add it as a broadcast kernel of its own
        return self._norm_act(_conv_pm(x, w, self.stride, self.padding), residual)

    def _norm_act(self, y: torch.Tensor, residual: Optional[torch.Tensor] = None, stats_ws: Optional[torch.Tensor] = None):
        """The norm, ReLU and residual join on the convolution's output y, in place."""
        if self.norm == "instance":
            if stats_ws is not None:
                return ops.instance_norm_apply(y, stats_ws, relu=self.relu, out=y)
            return ops.instance_norm_act(y, relu=self.relu, residual=residual, out=y)
        if self.norm == "group":  # the bias joins the statistics: a bias that differs within a group is not removed by its mean
            return ops.group_norm_act(y, self.gamma, self.beta, self.group, bias=self.bias, relu=self.relu, residual=residual,
                                      eps=self.eps, out=y, stats_ws=stats_ws)
        return ops.bias_act(y, self.bias, relu=self.relu, residual=residual, out=y)


class _Block(NamedTuple):
    """A residual block's steps: ``down`` the shortcut's convolution (None: identity), ``convs`` the branch in order; the one
    with ``residual`` set takes the join."""
    down: Optional[_EncConv]
    convs: List[_EncConv]


def _block(down: Optional[nn.Sequential], convs, dtype, device, native: Optional[str] = None, join: bool = True) -> _Block:
    """``down``: Sequential(1x1 convolution, norm) or None; ``convs``: the branch's (convolution, norm) pairs, each followed by
    ReLU; the last takes the residual join when ``join``."""
    last = len(convs) - 1
    return _Block(None if down is None else _EncConv(down[0], down[1], dtype, device, relu=False),
                  [_EncConv(c, n, dtype, device, residual=join and i == last, native=native) for i, (c, n) in enumerate(convs)])


def _run(blocks, x: torch.Tensor) -> torch.Tensor:
    for down, convs in blocks:
        xs = x if down is None else down(x)
        for step in convs:
            x = step(x, xs if step.residual else None)
    return x


class _Encoder(nn.Module):
    block = ResidualBlock
    widths = (64, 64, 96, 128)
    strides = (1, 2, 2)  # of layer1..3: output at 1/8
    project_shortcut = False  # ResidualBlock(project=True) in every block
    enc_conv3x3 = True  # the residual blocks' stride-1 3x3 convolutions on pfb_enc_conv3x3 where route_conv allows

    def __init__(self, output_dim: int = 128, norm_fn: str = "batch", dropout: float = 0.0) -> None:
        super().__init__()
        self.norm_fn = norm_fn
        w0, w1, w2, w3 = self.widths
        self.norm1 = _norm(norm_fn, w0, 8)
        self.conv1 = nn.Conv2d(3, w0, 7, stride=2, padding=3)
        self.relu1 = nn.ReLU(inplace=True)
        self.layer1 = self._stage(w0, w1, self.strides[0])
        self.layer2 = self._stage(w1, w2, self.strides[1])
        self.layer3 = self._stage(w2, w3, self.strides[2])
        self.conv2 = nn.Conv2d(w3, output_dim, 1)
        self.dropout = nn.Dropout2d(p=dropout) if dropout > 0 else None
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, (nn.BatchNorm2d, nn.InstanceNorm2d, nn.GroupNorm)) and m.weight is not None:
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def _stage(self, cin: int, cout: int, stride: int) -> nn.Sequential:
        kw = {"project": True} if self.project_shortcut else {}
        return nn.Sequential(self.block(cin, cout, self.norm_fn, stride=stride, **kw), self.block(cout, cout, self.norm_fn, stride=1, **kw))

    # ---- inference path: planned convolutions (_EncConv) on cuDNN and this library's kernels ----
    def _signature(self, dtype, device):
        return (dtype, str(device)) + tuple((p.data_ptr(), p._version) for p in self.parameters()) + \
            tuple((b.data_ptr(), b._version) for b in self.buffers())

    def _prepared(self, dtype, device):
        sig = self._signature(dtype, device)
        cache = getattr(self, "_prep_cache", None)
        if cache is not None and cache[0] == sig:
            return cache[1]
        with _prep_lock:  # several pipeline slots (host threads, streams) may arrive here together
            cache = getattr(self, "_prep_cache", None)
            if cache is not None and cache[0] == sig:
                return cache[1]
            plan = self._plan(dtype, device)
            # the fold / pack kernels ran on this thread's stream: finish them before other streams can see the cache
            torch.cuda.current_stream(device).synchronize()
            self._prep_cache = (sig, plan)
            return plan

    def _layers(self):
        """((first convolution, its norm), [(shortcut or None, [(convolution, norm), ...]) per block], output projection)."""
        blocks = []
        for blk in (*self.layer1, *self.layer2, *self.layer3):
            convs = [(blk.conv1, blk.norm1), (blk.conv2, blk.norm2)]
            blocks.append((blk.downsample, convs + [(blk.conv3, blk.norm3)] if isinstance(blk, BottleneckBlock) else convs))
        return (self.conv1, self.norm1), blocks, self.conv2

    def _plan(self, dtype, device):
        """(first convolution, output projection, blocks) as steps."""
        (conv1, norm1), blocks, proj = self._layers()
        native = "enc_conv3x3" if self.enc_conv3x3 else None
        return (_EncConv(conv1, norm1, dtype, device, native="first_conv7x7s2"),
                _EncConv(proj, None, dtype, device, relu=False, native="conv2d"),
                [_block(down, convs, dtype, device, native) for down, convs in blocks])

    def forward_pm(self, x: torch.Tensor) -> torch.Tensor:
        """x: pixel-major frames [N,H,W,3] on CUDA -> features [N,H/8,W/8,C] (H/4 with strides (1, 2, 1)) (eval semantics of
        extractor.py:171-194 / :246-267).  Batch norm is folded into the convolutions, instance norm + ReLU
        (+ residual join) is one fused pass (pfb_instance_norm_act) instead of five PyTorch kernels."""
        if self.norm_fn not in ("instance", "batch", "none"):
            return ops.to_pixel_major(self.forward(x.permute(0, 3, 1, 2)))
        first, proj, blocks = self._prepared(x.dtype, x.device)
        return proj(_run(blocks, first(x)))

    def forward(self, x):
        """Accepts one tensor or a list/tuple of two (processed as one batch: instance norm is
        per-sample, so this is exact -- extractor.py:173-176)."""
        pair = isinstance(x, (tuple, list))
        if pair:
            n = x[0].shape[0]
            x = torch.cat(list(x), dim=0)
        x = self.relu1(self.norm1(self.conv1(x)))
        x = self.layer3(self.layer2(self.layer1(x)))
        x = self.conv2(x)
        if self.training and self.dropout is not None:
            x = self.dropout(x)
        return (x[:n], x[n:]) if pair else x


class BasicEncoder(_Encoder):
    block = ResidualBlock
    widths = (64, 64, 96, 128)


class SmallEncoder(_Encoder):
    block = BottleneckBlock
    widths = (32, 32, 64, 96)
    enc_conv3x3 = False  # the bottlenecks stay on cuDNN
