"""CPU: the routes the encoders' plans give their convolutions (route_conv in models/raft/extractor.py), per storage type and
layer shape, and the ordered launches of every encoder against tests/golden/encoder_calls.npz.  Packing and launches are
shape-only fakes (tests/encoder_calls.py); the shape plan of pfb_enc_conv3x3 is host-only, so no device is needed."""
import pytest
import torch

import encoder_calls as E

NATIVE = {"first_conv7x7s2", "enc_conv3x3", "conv2d"}


@pytest.fixture(scope="module")
def ext():
    from ptlflow_b200.csrc import build as B
    from ptlflow_b200 import _lib
    from ptlflow_b200.models.raft import extractor

    import os
    if not os.path.exists(_lib.LIB_PATH):
        B.build()
    return extractor


def _steps(plan):
    if isinstance(plan, (list, tuple)):
        for p in plan:
            yield from _steps(p)
    elif plan is not None:
        yield plan


def _routes(enc, dtype):
    """{module name: route} over every convolution of the encoder's plan."""
    with E.fakes([]):
        plan = enc._prepared(dtype, torch.device("cpu"))
    names = {m: n for n, m in enc.named_modules()}
    return {names[s.conv]: s.route for s in _steps(plan)}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("norm", ["instance", "batch"])
def test_basic_encoder_routes_its_stride1_3x3_layers(ext, norm, dtype):
    enc = ext.BasicEncoder(output_dim=256, norm_fn=norm)
    routes = _routes(enc, dtype)
    expect = {"layer1.0.conv1", "layer1.0.conv2", "layer1.1.conv1", "layer1.1.conv2",  # 64 -> 64
              "layer3.0.conv2", "layer3.1.conv1", "layer3.1.conv2"}  # 128 -> 128
    if norm == "batch":  # 96 -> 96 only where bias, ReLU and the residual join go into the epilogue
        expect |= {"layer2.0.conv2", "layer2.1.conv2"}
    assert {n for n, r in routes.items() if r == "enc_conv3x3"} == expect
    # what stays off it: the 7x7 stride-2 first convolution and the output projection (kernels of their own), the stride-2
    # 3x3s and the 1x1 downsamples
    assert routes["conv1"] == "first_conv7x7s2" and routes["conv2"] == "conv2d"
    for n in ("layer2.0.conv1", "layer3.0.conv1", "layer2.0.downsample.0", "layer3.0.downsample.0"):
        assert routes[n] not in NATIVE, n


def test_fp32_stays_on_cudnn(ext):
    enc = ext.BasicEncoder(output_dim=256, norm_fn="instance")
    assert not NATIVE & set(_routes(enc, torch.float32).values())


def test_small_encoder_bottlenecks_stay_on_cudnn(ext):
    for dtype in (torch.float16, torch.bfloat16):
        enc = ext.SmallEncoder(output_dim=128, norm_fn="instance")
        assert "enc_conv3x3" not in _routes(enc, dtype).values()


def test_sea_raft_encoder_3x3_layers_stay_on_cudnn(ext):
    from ptlflow_b200.models.sea_raft.sea_raft import ResNetFPN

    enc = ResNetFPN((64, 96, 128), 64, "resnet18")  # 64 -> 64 and 128 -> 128 are shapes pfb_enc_conv3x3 runs
    routes = _routes(enc, torch.float16)
    assert "enc_conv3x3" not in routes.values()
    assert routes["conv1"] == "first_conv7x7s2" and routes["final_conv"] == "conv2d"


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
    route = lambda conv: ext.route_conv(conv, "batch", True, False, torch.float16, "enc_conv3x3")  # noqa: E731
    assert route(torch.nn.Conv2d(64, 64, 3, padding=1)) == "enc_conv3x3"
    for kw in (dict(padding=0), dict(padding=2, dilation=2), dict(padding=1, groups=2)):
        assert route(torch.nn.Conv2d(64, 64, 3, **kw)) == "cudnn_convolution_relu", kw


@pytest.fixture(scope="module")
def golden():
    return E.load_golden()


@pytest.mark.parametrize("key,model,net,dtype,channels,native", E.configs(), ids=[c[0] for c in E.configs()])
def test_encoder_launches_match_golden(ext, golden, key, model, net, dtype, channels, native):
    """fnet and cnet of every encoder family in fp32 / f16 / bf16 on 3- and 4-channel frames (and raft's f16 with
    PFB_NATIVE_ENC_CONV off): the same calls in the same order, with the same shapes, epilogues and operands."""
    assert E.record(model, net, dtype, channels, native) == golden[key]
