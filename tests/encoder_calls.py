"""What the encoders launch, recorded on the CPU: every launching function the inference path of the encoders calls is replaced
by a shape-only fake that logs one record per call and returns an empty tensor of the right shape.  ``record`` runs one
encoder's forward_pm (its preparation included) and returns the ordered records; tests/test_enc_conv_dispatch.py compares them
with tests/golden/encoder_calls.npz, which ``python tests/encoder_calls.py`` writes.  The library is needed only for
pfb_enc_conv3x3_supported (host side)."""
import contextlib
import copy
import functools
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden", "encoder_calls.npz")
MODELS = ["raft", "raft_small", "scv4", "scv8", "sea_raft_s", "sea_raft_m", "ms_raft_p", "ccmr", "ccmr_p"]
DTYPES = {"fp32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
BATCH, HEIGHT, WIDTH = 2, 64, 96  # frames per pair side; the grid is a multiple of 32 (ccmr's padding)


def _i(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _shape(t):
    return None if t is None else tuple(t.shape)


class _Packed:
    def __init__(self, cin, cout):
        self.Cin, self.Cout = cin, cout


@contextlib.contextmanager
def fakes(log):
    """Replaces the launching functions; each call appends (name, input dtype, input shape, output channels, epilogue, relu,
    bias passed, residual shape, stride, padding, statistics from conv1) to ``log``."""
    from ptlflow_b200 import ops

    def rec(name, x, cout=None, epi=None, relu=None, bias=None, res=None, stride=None, pad=None, stats=None):
        dt = None if x is None else str(x.dtype).replace("torch.", "")
        log.append(f"{name} {dt} in={_shape(x)} cout={cout} epi={epi} relu={relu} bias={bias} res={res} stride={stride} "
                   f"pad={pad} stats={stats}")

    def conv_out(x, w, stride, padding):  # x NCHW -> empty NCHW in channels_last, as cuDNN returns for channels_last input
        (sh, sw), (ph, pw) = _i(stride), _i(padding)
        n, _, h, wd = x.shape
        kh, kw = w.shape[2:]
        return torch.empty((n, w.shape[0], (h + 2 * ph - kh) // sh + 1, (wd + 2 * pw - kw) // sw + 1), dtype=x.dtype,
                           memory_format=torch.channels_last)

    def conv2d_cudnn(x, w, bias=None, stride=1, padding=0, dilation=1, groups=1):
        rec("F.conv2d", x, w.shape[0], bias=bias is not None, stride=_i(stride), pad=_i(padding))
        return conv_out(x, w, stride, padding)

    def cudnn_convolution_relu(x, w, bias, stride, padding, dilation, groups):
        rec("cudnn_convolution_relu", x, w.shape[0], relu=True, bias=bias is not None, stride=_i(stride), pad=_i(padding))
        return conv_out(x, w, stride, padding)

    def enc_conv3x3(x, packed, epilogue=0, bias=None, residual=None, out=None, out_offset=0):
        rec("enc_conv3x3", x, packed.Cout, epilogue, bias=bias is not None, res=_shape(residual))
        return torch.empty(tuple(x.shape[:3]) + (packed.Cout,), dtype=x.dtype)

    def first_conv7x7s2(x, wpack, bias, relu, stats_ws=None):
        rec("first_conv7x7s2", x, 64, relu=relu, bias=bias is not None, stats=stats_ws is not None)
        n, h, w, _ = x.shape
        return torch.empty((n, h // 2, w // 2, 64), dtype=x.dtype)

    def instance_norm_act(x, relu=True, residual=None, eps=1e-5, out=None):
        rec("instance_norm_act", x, relu=relu, res=_shape(residual))
        return out if out is not None else torch.empty_like(x)

    def instance_norm_apply(x, ws, relu=True, residual=None, eps=1e-5, out=None):
        rec("instance_norm_apply", x, relu=relu, res=_shape(residual), stats=True)
        return out if out is not None else torch.empty_like(x)

    def instance_norm_workspace(x_shape, device):
        rec("instance_norm_workspace", None, x_shape[-1])
        return torch.empty(3 * x_shape[0] * x_shape[-1], dtype=torch.float64)

    def bias_act(x, bias, relu=True, residual=None, out=None):
        rec("bias_act", x, relu=relu, bias=bias is not None, res=_shape(residual))
        return out if out is not None else torch.empty_like(x)

    def group_norm_act(x, gamma, beta, group_size, bias=None, relu=True, residual=None, eps=1e-5, out=None, stats_ws=None):
        rec("group_norm_act", x, epi=group_size, relu=relu, bias=bias is not None, res=_shape(residual), stats=stats_ws is not None)
        return out if out is not None else torch.empty_like(x)

    def upsample2x_concat(src, skip, out=None):
        rec("upsample2x_concat", src, src.shape[-1] + (0 if skip is None else skip.shape[-1]), res=_shape(skip))
        b, h, w, c = src.shape
        return torch.empty((b, 2 * h, 2 * w, c + (0 if skip is None else skip.shape[-1])), dtype=src.dtype)

    def conv2d(srcs, packed, out, epilogue=0, **kw):
        rec("ops.conv2d", srcs[0], packed.Cout, epilogue, res=_shape(out))
        return out

    def packed_conv(convs, dtype, device, cout_align=8, src_channels=None):
        w = convs[0].weight
        rec("PackedConv", w, sum(c.weight.shape[0] for c in convs), bias=convs[0].bias is not None, res=src_channels,
            stats=str(dtype).replace("torch.", ""))
        return _Packed(w.shape[1], sum(c.weight.shape[0] for c in convs))

    def pack_first_conv(weight, dtype):
        rec("pack_first_conv", weight, weight.shape[0], stats=str(dtype).replace("torch.", ""))
        return torch.empty((9, 16, 4, 8, 8), dtype=dtype)

    class _Stream:
        def synchronize(self):
            rec("synchronize", None)

    def current_stream(device=None):
        return _Stream()

    swaps = [(ops, n, f) for n, f in (("enc_conv3x3", enc_conv3x3), ("first_conv7x7s2", first_conv7x7s2),
                                      ("instance_norm_act", instance_norm_act), ("instance_norm_apply", instance_norm_apply),
                                      ("instance_norm_workspace", instance_norm_workspace), ("bias_act", bias_act),
                                      ("group_norm_act", group_norm_act), ("upsample2x_concat", upsample2x_concat),
                                      ("conv2d", conv2d), ("PackedConv", packed_conv), ("pack_first_conv", pack_first_conv))]
    swaps += [(F, "conv2d", conv2d_cudnn), (torch, "cudnn_convolution_relu", cudnn_convolution_relu),
              (torch.cuda, "current_stream", current_stream)]
    saved = [(m, n, getattr(m, n)) for m, n, _ in swaps]
    try:
        for m, n, f in swaps:
            setattr(m, n, f)
        yield log
    finally:
        for m, n, f in saved:
            setattr(m, n, f)


def load_golden():
    """{configuration key: ordered records} of tests/golden/encoder_calls.npz."""
    out = {}
    for part in bytes(np.load(GOLDEN)["calls"]).decode().split("# ")[1:]:
        key, *log = part.rstrip("\n").split("\n")
        out[key] = log
    return out


def configs():
    """(key, model, encoder, dtype name, frame channels, native enc_conv3x3)."""
    out = [(m, net, dt, ch, True) for m in MODELS for dt in DTYPES for ch in (3, 4) for net in ("fnet", "cnet")]
    out += [("raft", net, "f16", ch, False) for ch in (3, 4) for net in ("fnet", "cnet")]
    return [(f"{m}.{net}.{dt}.c{ch}" + ("" if native else ".cudnn_enc"), m, net, dt, ch, native) for m, net, dt, ch, native in out]


@functools.lru_cache(maxsize=None)
def _encoder(model, net, dtype):
    import ptlflow_b200 as pb

    torch.manual_seed(0)
    return getattr(pb.get_model(model), net).eval().to(DTYPES[dtype])


def record(model, net, dtype, channels, native_enc_conv=True):
    """The ordered records of one forward_pm of ``model``'s ``net`` ('fnet' or 'cnet'), as RAFT._encode feeds it: fnet both
    frames of the pairs, cnet the first frames (SEA-RAFT's cnet: both frames' RGB side by side)."""
    from ptlflow_b200.models.raft import extractor

    dt = DTYPES[dtype]
    enc = copy.deepcopy(_encoder(model, net, dtype))  # a fresh copy prepares again
    frames = torch.zeros((2 * BATCH, HEIGHT, WIDTH, channels), dtype=dt)
    x = frames if net == "fnet" else frames[:BATCH]
    if net == "cnet" and enc.conv1.in_channels == 6:
        x = torch.cat([frames[:BATCH, ..., :3], frames[BATCH:, ..., :3]], dim=-1)
    log = []
    saved = extractor._NATIVE_ENC_CONV
    extractor._NATIVE_ENC_CONV = native_enc_conv
    try:
        with torch.no_grad(), fakes(log):
            enc.forward_pm(x)
    finally:
        extractor._NATIVE_ENC_CONV = saved
    return log


def main():
    from ptlflow_b200 import _lib
    from ptlflow_b200.csrc import build

    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    calls = {key: record(*cfg) for key, *cfg in configs()}
    text = "".join(f"# {key}\n" + "".join(rec + "\n" for rec in log) for key, log in calls.items())
    np.savez_compressed(GOLDEN, calls=np.frombuffer(text.encode(), dtype=np.uint8))
    print(f"{GOLDEN}: {len(calls)} configurations, {sum(len(log) for log in calls.values())} calls")


if __name__ == "__main__":
    main()
