"""CPU: which encoder convolutions the dispatch of models/raft/extractor.py routes to pfb_enc_conv3x3, per storage type and
layer shape.  The eligibility predicate is host-only (the shape plan of csrc/enc_conv_umma.cu), so no device is needed."""
import pytest
import torch


@pytest.fixture(scope="module")
def ext():
    from ptlflow_b200.csrc import build as B
    from ptlflow_b200 import _lib
    from ptlflow_b200.models.raft import extractor

    import os
    if not os.path.exists(_lib.LIB_PATH):
        B.build()
    return extractor


def _routed(enc, dtype, ext):
    """{module name: routed} over every convolution of the encoder, as _Encoder._prepare_locked decides (a residual block's
    conv2 takes its residual join into the kernel unless an instance norm sits between)."""
    return {name: ext.enc_conv_eligible(m, dtype, fused_residual=name.endswith(".conv2") and enc.norm_fn != "instance")
            for name, m in enc.named_modules() if isinstance(m, torch.nn.Conv2d)}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("norm", ["instance", "batch"])
def test_basic_encoder_routes_its_stride1_3x3_layers(ext, norm, dtype):
    enc = ext.BasicEncoder(output_dim=256, norm_fn=norm)
    routed = _routed(enc, dtype, ext)
    expect = {"layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv1", "layer1.1.conv2",  # 64 -> 64
              "layer3.0.conv2", "layer3.1.conv1", "layer3.1.conv2"}  # 128 -> 128
    if norm == "batch":  # 96 -> 96 only where bias, ReLU and the residual join go into the epilogue
        expect |= {"layer2.0.conv2", "layer2.1.conv2"}
    assert {n for n, r in routed.items() if r} == expect
    # what stays on cuDNN: the 7x7 stride-2 first convolution (its own kernel), the stride-2 3x3s, the 1x1 downsamples and
    # the output projection
    for n in ("conv1", "layer2.0.conv1", "layer3.0.conv1", "layer2.0.downsample.0", "layer3.0.downsample.0", "conv2"):
        assert not routed[n], n


def test_fp32_stays_on_cudnn(ext):
    enc = ext.BasicEncoder(output_dim=256, norm_fn="instance")
    assert not any(_routed(enc, torch.float32, ext).values())


def test_small_encoder_bottlenecks_stay_on_cudnn(ext):
    for dtype in (torch.float16, torch.bfloat16):
        enc = ext.SmallEncoder(output_dim=128, norm_fn="instance")
        assert not any(_routed(enc, dtype, ext).values())


def test_supported_channel_counts(ext):
    from ptlflow_b200 import ops

    for dtype in (torch.float16, torch.bfloat16):
        for cin in (32, 64, 96, 128, 192, 256):
            for cout in (64, 96, 128):
                assert ops.enc_conv3x3_supported(cin, cout, dtype), (cin, cout, dtype)
        for cin, cout in ((16, 64), (48, 64), (64, 32), (64, 48), (64, 160), (64, 256)):
            assert not ops.enc_conv3x3_supported(cin, cout, dtype), (cin, cout, dtype)
    assert not ops.enc_conv3x3_supported(64, 64, torch.float32)
    # a 3x3 with padding 0, a dilated one and a grouped one are not the kernel's convolution
    for kw in (dict(padding=0), dict(padding=2, dilation=2), dict(padding=1, groups=2)):
        assert not ext.enc_conv_eligible(torch.nn.Conv2d(64, 64, 3, **kw), torch.float16), kw
