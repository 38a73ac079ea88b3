"""Conformance of the encoders' 3x3 stride-1 convolution (pfb_enc_conv3x3, csrc/enc_conv_umma.cu) against a float64 reference,
element by element, with the per-element bound of conv_reference.py.

The sweep covers f16 and bf16, every (Cin, Cout) in {64, 96, 128}^2 and a 32-channel input, the three epilogues, batches of 1
and 3, and ragged grids whose partial work items (the last 256- or 128-pixel row piece, a second warpgroup beyond the right
edge) and halos touch every border; plus the config-2 layer1 shape (220 x 512, 64 -> 64).  Outputs are written into a wider
sentinel-filled buffer at a channel offset with spare pixels behind it: nothing outside the layer's channels and pixels may
change.  The two context-encoder epilogues are written here in float64:

    BIAS_RELU           relu(acc + bias)
    BIAS_RELU_RESIDUAL  relu(res + relu(acc + bias))

relu is 1-Lipschitz, so the accumulator bound E of conv_reference carries through; the residual add is one more fp32
rounding of a value bounded by |res| + S."""
import zlib

import pytest
import torch

import conv_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HALF = [torch.float16, torch.bfloat16]
LINEAR, BIAS_RELU, BIAS_RELU_RESIDUAL = range(3)  # pfb_enc_conv_epilogue
EPIS = {LINEAR: "linear", BIAS_RELU: "bias_relu", BIAS_RELU_RESIDUAL: "bias_relu_residual"}


def _seed(*parts):
    return zlib.crc32("/".join(str(p) for p in parts).encode())


def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV) * scale


class _Conv(torch.nn.Module):
    def __init__(self, weight):
        super().__init__()
        self.weight, self.bias = weight, None


def reference(epi, acc, S, n, dtype, residual=None):
    """(ref, bound) of an epilogue in float64."""
    rho, eta = R.RHO[dtype], R.ETA[dtype]
    E = (n + R.C_SPARE) * R.U * S
    if epi == LINEAR:
        ref, err = acc, E
    elif epi == BIAS_RELU:
        ref, err = acc.clamp_min(0.0), E
    else:
        r = residual.double()
        ref = (r + acc.clamp_min(0.0)).clamp_min(0.0)
        err = E + R.U * (r.abs() + S)
    return ref, rho * ref.abs() + (1.0 + rho) * err + eta


def run(B, H, W, cin, cout, epi, dtype, out_offset=8):
    from ptlflow_b200 import ops

    sd = _seed(B, H, W, cin, cout, epi)
    x = _randn((B, H, W, cin), sd).to(dtype)
    w = _randn((cout, cin, 3, 3), sd + 1, (9 * cin) ** -0.5)
    bias = _randn((cout,), sd + 2, 0.3)
    packed = ops.PackedConv([_Conv(w)], dtype, DEV, src_channels=[cin])
    res = _randn((B, H, W, cout), sd + 3).to(dtype) if epi == BIAS_RELU_RESIDUAL else None
    acc, S, n = R.conv_terms([x.double()], R.q(w, dtype), None if epi == LINEAR else bias.double())
    ref, bound = reference(epi, acc, S, n, dtype, res)

    stride = out_offset + cout + 8
    numel = B * H * W * stride
    base = torch.full((numel + 64 * stride,), R.SENTINEL, dtype=dtype, device=DEV)  # spare pixels behind the output
    out = base[:numel].view(B, H, W, stride)
    before = base.clone()
    ops.enc_conv3x3(x, packed, epi, bias=None if epi == LINEAR else bias, residual=res, out=out, out_offset=out_offset)
    torch.cuda.synchronize()
    what = f"B={B} {H}x{W} {cin}->{cout} {EPIS[epi]} {dtype}"
    worst = R.assert_within(out[..., out_offset:out_offset + cout], ref, bound, what=what)
    R.assert_untouched(out, before[:numel].view(B, H, W, stride), out_offset, out_offset + cout, what=what)
    assert torch.equal(R.bits(base[numel:]), R.bits(before[numel:])), f"{what}: pixels behind the output were written"
    return worst


CHANNELS = [(ci, co) for ci in (64, 96, 128) for co in (64, 96, 128)] + [(32, 64), (32, 96), (32, 128)]
# ragged grids: the last row piece partial for both tile widths (301 = 256 + 45 = 2 * 128 + 45), a second warpgroup wholly
# beyond the right edge (Cout 64 on 37 or 130 pixels), one-row and one-pixel-wide images
GRIDS = [(1, 7, 301), (3, 5, 37), (1, 1, 130), (3, 9, 1)]


@pytest.mark.parametrize("dtype", HALF, ids=["f16", "bf16"])
@pytest.mark.parametrize("epi", list(EPIS), ids=list(EPIS.values()))
@pytest.mark.parametrize("cin,cout", CHANNELS, ids=[f"{a}x{b}" for a, b in CHANNELS])
def test_enc_conv_shapes(cin, cout, epi, dtype):
    for B, H, W in GRIDS:
        run(B, H, W, cin, cout, epi, dtype)


@pytest.mark.parametrize("dtype", HALF, ids=["f16", "bf16"])
@pytest.mark.parametrize("epi", list(EPIS), ids=list(EPIS.values()))
def test_enc_conv_config2_layer1(epi, dtype):
    """RAFT's layer1 at 1024 x 436 (padded to 440): a 220 x 512 grid, 64 -> 64 channels, contiguous output."""
    run(3, 220, 512, 64, 64, epi, dtype, out_offset=0)


def test_enc_conv_rejects_bad_arguments():
    from ptlflow_b200 import _lib, ops

    x = torch.zeros((1, 4, 8, 64), dtype=torch.float16, device=DEV)
    packed = ops.PackedConv([_Conv(torch.zeros((48, 64, 3, 3), device=DEV))], torch.float16, DEV, src_channels=[64])
    with pytest.raises(RuntimeError, match="unsupported shape"):
        ops.enc_conv3x3(x, packed)  # Cout 48
    packed = ops.PackedConv([_Conv(torch.zeros((64, 64, 3, 3), device=DEV))], torch.float16, DEV, src_channels=[64])
    with pytest.raises(RuntimeError, match="needs a bias"):
        ops.enc_conv3x3(x, packed, _lib.ENC_CONV_BIAS_RELU)
