"""Feature / context encoders (SURVEY.md 8(a) row a14: not on the named hot path, kept as
cuDNN modules in channels_last; parameter names and shapes equal the reference's
ptlflow/models/raft/extractor.py:122-267 so checkpoints load strictly)."""
from __future__ import annotations

import os
import threading

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


def _fold(conv: nn.Conv2d, norm: nn.Module, dtype, device):
    """(weight, bias) of ``conv`` in channels_last storage; an eval-mode BatchNorm that follows is folded in
    (y = s * conv(x) + t  ->  weight * s, bias * s + t).  Instance norm / identity leave the conv as is."""
    w = conv.weight.detach().to(device=device, dtype=torch.float32)
    b = conv.bias.detach().to(device=device, dtype=torch.float32) if conv.bias is not None else torch.zeros(w.shape[0], device=device)
    if isinstance(norm, nn.BatchNorm2d):
        s = norm.weight.detach().float().to(device) / torch.sqrt(norm.running_var.detach().float().to(device) + norm.eps)
        t = norm.bias.detach().float().to(device) - norm.running_mean.detach().float().to(device) * s
        w = w * s.view(-1, 1, 1, 1)
        b = b * s + t
    w = w.to(dtype).contiguous(memory_format=torch.channels_last)
    b = b.contiguous()  # fp32: added by this library's kernels
    if dtype == torch.float32:
        return w, b
    return w, b, b.to(dtype)  # + the storage-type copy cuDNN's fused bias + ReLU epilogue wants (cast once, not per forward)


_NATIVE_CONV1 = bool(int(os.environ.get("PFB_NATIVE_CONV1", "1")))
_NATIVE_CONV2 = bool(int(os.environ.get("PFB_NATIVE_CONV2", "1")))
# the residual blocks' 3x3 stride-1 convolutions on pfb_enc_conv3x3 (read at every forward: tools/time_encoder_convs.py
# switches it to compare both paths in one process)
_NATIVE_ENC_CONV = bool(int(os.environ.get("PFB_NATIVE_ENC_CONV", "1")))
# (Cin, Cout) of eligible layers that stay on cuDNN unless the kernel also takes their residual join: at 96 output channels
# the kernel computes 128 MMA rows, and cuDNN measured faster on the plain convolution (DESIGN.md section 5)
_ENC_CONV_CUDNN_UNFUSED = frozenset({(96, 96)})
# batch-norm-folded convolutions without a residual join: cuDNN's own conv + bias + ReLU epilogue instead of a separate pass
_CUDNN_FUSED_RELU = bool(int(os.environ.get("PFB_CUDNN_FUSED_RELU", "1")))
_prep_lock = threading.Lock()


def _conv_pm(x: torch.Tensor, wb, stride: int, padding: int) -> torch.Tensor:
    """cuDNN convolution on a pixel-major tensor [N,H,W,C] -> [N,H',W',C'] (channels_last in and out, no copies)."""
    # no bias here: PyTorch would add it as a separate broadcast kernel; it is folded into pfb_bias_act (batch / no norm)
    # and is mathematically irrelevant in front of an instance norm (a per-channel constant is removed by the mean)
    y = F.conv2d(x.permute(0, 3, 1, 2), wb[0], None, stride=stride, padding=padding)
    y = y.permute(0, 2, 3, 1)
    return y if y.is_contiguous() else y.contiguous()


def enc_conv_eligible(conv: nn.Conv2d, dtype: torch.dtype, fused_residual: bool = False) -> bool:
    """A 3x3 stride-1 "same" convolution that pfb_enc_conv3x3 runs in this storage type (f16 / bf16; Cin a multiple of 32,
    Cout 64, 96 or 128), and that cuDNN did not measure faster on.  ``fused_residual``: the layer's bias, ReLU and residual
    join would go into the kernel's epilogue (a batch-norm-folded block's second convolution)."""
    return (tuple(conv.kernel_size) == (3, 3) and tuple(conv.stride) == (1, 1) and tuple(conv.padding) == (1, 1)
            and tuple(conv.dilation) == (1, 1) and conv.groups == 1 and conv.padding_mode == "zeros"
            and (fused_residual or (conv.in_channels, conv.out_channels) not in _ENC_CONV_CUDNN_UNFUSED)
            and ops.enc_conv3x3_supported(conv.in_channels, conv.out_channels, dtype))


class _Encoder(nn.Module):
    block = ResidualBlock
    widths = (64, 64, 96, 128)
    strides = (1, 2, 2)  # of layer1..3: output at 1/8
    project_shortcut = False  # ResidualBlock(project=True) in every block

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

    # ---- inference path: cuDNN convs + this library's fused norm / activation / residual kernels ----
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
            return self._prepare_locked(sig, dtype, device)

    def _prepare_locked(self, sig, dtype, device):
        prep = {"conv1": _fold(self.conv1, self.norm1, dtype, device), "conv2": _fold(self.conv2, nn.Identity(), dtype, device), "blocks": []}
        for layer in (self.layer1, self.layer2, self.layer3):
            for blk in layer:
                e = {"stride": blk.conv2.stride[0] if isinstance(blk, BottleneckBlock) else blk.conv1.stride[0]}
                names = ("conv1", "conv2", "conv3") if isinstance(blk, BottleneckBlock) else ("conv1", "conv2")
                for i, nme in enumerate(names, start=1):
                    e[nme] = _fold(getattr(blk, nme), getattr(blk, f"norm{i}"), dtype, device)
                if blk.downsample is not None:
                    e["down"] = _fold(blk.downsample[0], blk.downsample[1], dtype, device)
                prep["blocks"].append(e)
        if (_NATIVE_CONV1 and tuple(self.conv1.weight.shape) == (64, 3, 7, 7) and dtype in (torch.float16, torch.bfloat16)
                and self.norm_fn in ("instance", "batch", "none")):
            folded = _fold(self.conv1, self.norm1, torch.float32, device)
            prep["conv1_native"] = (ops.pack_first_conv(folded[0], dtype), folded[1])
        # the output projection (1x1, w3 -> output_dim) on this library's wgmma implicit-GEMM kernel with the bias in its
        # epilogue: cuDNN picked an sm_80 kernel without shared-memory staging for it (50 us per encoder, ncu launch list r02f)
        # and the bias needed a pass of its own
        c2 = self.conv2
        if (_NATIVE_CONV2 and dtype in (torch.float16, torch.bfloat16) and tuple(c2.kernel_size) == (1, 1) and c2.in_channels % 64 == 0
                and c2.out_channels % 32 == 0 and c2.out_channels <= 1024):
            prep["conv2_native"] = ops.PackedConv([c2], dtype, device, src_channels=[c2.in_channels])
        # the residual blocks' 3x3 stride-1 convolutions on pfb_enc_conv3x3 (output channels on the MMA's M dimension): packed
        # from the folded fp32 weights (rounded to the storage type once, as _fold does for cuDNN), with the fp32 bias.  Packed
        # whatever PFB_NATIVE_ENC_CONV says: forward_pm reads the switch at every call
        if dtype in (torch.float16, torch.bfloat16):
            blocks = [blk for layer in (self.layer1, self.layer2, self.layer3) for blk in layer]
            for e, blk in zip(prep["blocks"], blocks):
                if not isinstance(blk, ResidualBlock):
                    continue
                for nme, norm in (("conv1", blk.norm1), ("conv2", blk.norm2)):
                    conv = getattr(blk, nme)
                    if enc_conv_eligible(conv, dtype, fused_residual=nme == "conv2" and self.norm_fn != "instance"):
                        w, b = _fold(conv, norm, torch.float32, device)
                        e[nme + "_enc"] = (ops.PackedConv([ops.ConvWeights(w)], dtype, device, src_channels=[conv.in_channels]), b)
        # the fold / pack kernels ran on this thread's stream: finish them before other streams can see the cache
        torch.cuda.current_stream(device).synchronize()
        self._prep_cache = (sig, prep)
        return prep

    def forward_pm(self, x: torch.Tensor) -> torch.Tensor:
        """x: pixel-major frames [N,H,W,3] on CUDA -> features [N,H/8,W/8,C] (H/4 with strides (1, 2, 1)) (eval semantics of
        extractor.py:171-194 / :246-267).  Batch norm is folded into the convolutions, instance norm + ReLU
        (+ residual join) is one fused pass (pfb_instance_norm_act) instead of five PyTorch kernels."""
        if self.norm_fn not in ("instance", "batch", "none"):
            return ops.to_pixel_major(self.forward(x.permute(0, 3, 1, 2)))
        inst = self.norm_fn == "instance"
        prep = self._prepared(x.dtype, x.device)

        def conv_act(x, wb, stride, padding, relu=True, residual=None, native=None):
            if (native is not None and _NATIVE_ENC_CONV and relu and x.is_contiguous()
                    and (residual is None or residual.is_contiguous())):
                packed, bias = native
                if inst:  # the instance norm removes the bias
                    y = ops.enc_conv3x3(x, packed)
                    return ops.instance_norm_act(y, relu=True, residual=residual, out=y)
                epi = _lib.ENC_CONV_BIAS_RELU if residual is None else _lib.ENC_CONV_BIAS_RELU_RESIDUAL
                return ops.enc_conv3x3(x, packed, epi, bias=bias, residual=residual)
            if _CUDNN_FUSED_RELU and not inst and relu and residual is None and x.dtype != torch.float32:
                bh = wb[2] if len(wb) > 2 else wb[1].to(x.dtype)
                y = torch.cudnn_convolution_relu(x.permute(0, 3, 1, 2), wb[0], bh, (stride, stride), (padding, padding), (1, 1), 1)
                y = y.permute(0, 2, 3, 1)
                return y if y.is_contiguous() else y.contiguous()
            y = _conv_pm(x, wb, stride, padding)
            if inst:
                return ops.instance_norm_act(y, relu=relu, residual=residual, out=y)
            return ops.bias_act(y, wb[1], relu=relu, residual=residual, out=y)

        c1 = prep["conv1"]
        native_c1 = ("conv1_native" in prep and x.shape[-1] == 4 and tuple(self.conv1.weight.shape) == (64, 3, 7, 7) and x.dtype in (torch.float16, torch.bfloat16)
                     and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0)
        if native_c1:
            # wgmma first convolution (csrc/first_conv.cu): statistics of the instance norm come out of its epilogue,
            # bias + ReLU of the folded batch norm are applied in it
            wpack, bias = prep["conv1_native"]
            if inst:
                ws = ops.instance_norm_workspace((x.shape[0], 0, 0, 64), x.device)
                y = ops.first_conv7x7s2(x, wpack, None, relu=False, stats_ws=ws)
                x = ops.instance_norm_apply(y, ws, relu=True, out=y)
            else:
                x = ops.first_conv7x7s2(x, wpack, bias, relu=True)
        elif x.shape[-1] != c1[0].shape[1]:  # frames carry zero channels beyond RGB (8-byte pixels): pad the filter to match
            key = ("conv1_pad", x.shape[-1])
            if key not in prep:
                w = torch.zeros((c1[0].shape[0], x.shape[-1]) + tuple(c1[0].shape[2:]), dtype=c1[0].dtype, device=c1[0].device)
                w[:, : c1[0].shape[1]] = c1[0]
                prep[key] = (w.contiguous(memory_format=torch.channels_last), c1[1])
            c1 = prep[key]
        if not native_c1:
            x = conv_act(x, c1, 2, 3)
        for e in prep["blocks"]:
            s = e["stride"]
            xs = conv_act(x, e["down"], s, 0, relu=False) if "down" in e else x
            if "conv3" in e:  # bottleneck: 1x1 -> 3x3 (stride) -> 1x1
                y = conv_act(x, e["conv1"], 1, 0)
                y = conv_act(y, e["conv2"], s, 1)
                x = conv_act(y, e["conv3"], 1, 0, relu=True, residual=xs)
            else:  # residual: 3x3 (stride) -> 3x3
                y = conv_act(x, e["conv1"], s, 1, native=e.get("conv1_enc"))
                x = conv_act(y, e["conv2"], 1, 1, relu=True, residual=xs, native=e.get("conv2_enc"))
        if "conv2_native" in prep and x.is_contiguous():
            packed = prep["conv2_native"]
            out = torch.empty(x.shape[:3] + (packed.Cout,), dtype=x.dtype, device=x.device)
            return ops.conv2d([x], packed, out, epilogue=_lib.EPI_LINEAR)
        y = _conv_pm(x, prep["conv2"], 1, 0)
        return ops.bias_act(y, prep["conv2"][1], relu=False, out=y)

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
