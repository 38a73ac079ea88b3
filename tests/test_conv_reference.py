"""The float64 convolution reference and its per-element bound (conv_reference.py) on the CPU: the reference rounded once to
the storage type passes, and each of a set of plausible kernel bugs, planted into the float64 result of a small case, is
rejected, in f16 and in bf16.  This is what makes "the conformance tests would fail if the kernel were subtly wrong" a
tested property."""
import math

import pytest
import torch

import conv_reference as R

DTYPES = [torch.float16, torch.bfloat16]
B, H, W, KH, KW = 1, 5, 20, 3, 3
CHANS = [80, 48]      # source 0 ends in a partial 64-channel chunk (channels 64..79)
COUT, NT, TW = 192, 96, 16   # two N tiles of 96 columns; M tiles 16 pixels wide


def _gen(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64) * scale


def _inputs(dtype, cout=COUT, chans=CHANS, kh=KH, kw=KW, seed=0):
    cin = sum(chans)
    xs = [R.q(_gen((B, H, W, c), seed + i), dtype) for i, c in enumerate(chans)]
    w = R.q(_gen((cout, cin, kh, kw), seed + 10, 1.0 / math.sqrt(cin * kh * kw)), dtype)
    bias = R.q(_gen((cout,), seed + 11, 0.1), torch.float32)
    return xs, w, bias


def _tap_only(w, ky, kx):
    m = torch.zeros_like(w)
    m[:, :, ky, kx] = w[:, :, ky, kx]
    return m


def _planted(fault, dtype):
    """(reference out, bound, out with the fault) for a LINEAR layer with scale 0.75."""
    xs, w, bias = _inputs(dtype)
    acc, S, n = R.conv_terms(xs, w, bias)
    bad = acc.clone()
    if fault == "tap_dropped_in_one_tile_row":
        contrib, _, _ = R.conv_terms(xs, _tap_only(w, 0, 1))
        bad[:, 2, :TW] -= contrib[:, 2, :TW]
    elif fault == "halo_shifted_at_tile_edge":
        bad[:, :, TW - 1] = acc[:, :, TW]  # the last column of the first M tile reads its taps one pixel to the right
    elif fault == "partial_chunk_dropped":
        wd = w.clone()
        wd[:, 64:80] = 0
        bad, _, _ = R.conv_terms(xs, wd, bias)
    elif fault == "chunk_from_neighbour_n_tile":
        bad[..., 0:32] = acc[..., NT:NT + 32]
    elif fault == "bias_added_twice":
        bad = acc + bias
    else:
        raise ValueError(fault)
    ref, bound = R.epilogue(R.LINEAR, acc, S, n, dtype, scale=0.75)["out"]
    got, _ = R.epilogue(R.LINEAR, bad, S, n, dtype, scale=0.75)["out"]
    return ref, bound, R.q(got, dtype)


FAULTS = ["tap_dropped_in_one_tile_row", "halo_shifted_at_tile_edge", "partial_chunk_dropped", "chunk_from_neighbour_n_tile",
          "bias_added_twice"]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
@pytest.mark.parametrize("fault", FAULTS)
def test_bound_rejects_planted_fault(fault, dtype):
    ref, bound, got = _planted(fault, dtype)
    assert R.within(R.q(ref, dtype), ref, bound)
    assert not R.within(got, ref, bound), fault


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_bound_rejects_missing_flow_columns(dtype):
    xs, w, bias = _inputs(dtype, cout=126)
    acc, S, n = R.conv_terms(xs, w, bias)
    flow = R.q(_gen((B, H, W, 2), 5, 3.0), torch.float32)
    for epi in (R.RELU_APPEND_FLOW, R.LINEAR_APPEND_FLOW):
        ref, bound = R.epilogue(epi, acc, S, n, dtype, flow=flow)["out"]
        assert ref.shape[-1] == 128
        got = R.q(ref, dtype)
        assert R.within(got, ref, bound)
        got[..., 126:] = 0
        assert not R.within(got, ref, bound)
        got[..., 126:] = R.SENTINEL
        assert not R.within(got, ref, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_bound_rejects_swapped_gate_operands(dtype):
    hd = 64
    xs, w, bias = _inputs(dtype, cout=hd, chans=[64, 64])
    acc, S, n = R.conv_terms(xs, w, bias)
    h = R.q(torch.tanh(_gen((B, H, W, hd), 6)), dtype)
    z = R.q(torch.sigmoid(_gen((B, H, W, hd), 7)), dtype)
    ref, bound = R.epilogue(R.GRU_Q, acc, S, n, dtype, h=h, z=z, hidden=hd)["out"]
    assert R.within(R.q(ref, dtype), ref, bound)
    swapped, _ = R.epilogue(R.GRU_Q, acc, S, n, dtype, h=z, z=h, hidden=hd)["out"]
    assert not R.within(R.q(swapped, dtype), ref, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f16", "bf16"])
def test_rounded_reference_passes_every_epilogue(dtype):
    """The unperturbed reference, rounded once to the storage type, is inside the bound for every epilogue."""
    hd = 64
    xs, w, bias = _inputs(dtype, cout=2 * hd, chans=[64, 48])
    acc, S, n = R.conv_terms(xs, w, bias)
    h = R.q(torch.tanh(_gen((B, H, W, 2 * hd), 8)), dtype)
    z = R.q(torch.sigmoid(_gen((B, H, W, 2 * hd), 9)), dtype)
    res = R.q(_gen((B, H, W, 2 * hd), 12), dtype)
    pw, pb = R.q(_gen((2 * hd,), 13, 0.5), torch.float32), R.q(_gen((2 * hd,), 14, 0.1), torch.float32)
    flow = R.q(_gen((B, H, W, 2), 15, 3.0), torch.float32)
    cases = {
        "linear": (R.LINEAR, dict(scale=0.3)), "relu": (R.RELU, {}), "gelu": (R.GELU, {}), "axpy": (R.AXPY, dict(h=h, scale=-0.7)),
        "residual_gelu": (R.RESIDUAL_GELU, dict(residual=res)), "residual_gelu_post": (R.RESIDUAL_GELU, dict(residual=res, post_w=pw, post_b=pb)),
        "gru_zr": (R.GRU_ZR, dict(h=h[..., :hd], hidden=hd)), "relu_append_flow": (R.RELU_APPEND_FLOW, dict(flow=flow)),
    }
    for name, (epi, kw) in cases.items():
        for key, (ref, bound) in R.epilogue(epi, acc, S, n, dtype, **kw).items():
            assert R.within(R.q(ref, dtype), ref, bound), (name, key)
    ref, bound = R.epilogue(R.LINEAR_F32, acc, S, n, torch.float32, scale=0.3)["out"]
    assert R.within(ref.float(), ref, bound)
    ref, bound = R.epilogue(R.GRU_Q, acc[..., :hd], S[..., :hd], n, dtype, h=h[..., :hd], z=z[..., :hd], hidden=hd)["out"]
    assert R.within(R.q(ref, dtype), ref, bound)


def test_sentinel_check_sees_stray_writes():
    buf = torch.full((2, 3, 4, 40), R.SENTINEL, dtype=torch.float16)
    before = buf.clone()
    buf[..., 8:36] = 1.0
    R.assert_untouched(buf, before, 8, 36)
    buf[0, 1, 2, 36] = 0.0
    with pytest.raises(AssertionError):
        R.assert_untouched(buf, before, 8, 36)


def test_ratio_flags_non_finite_output():
    ref = torch.ones(4, dtype=torch.float64)
    bound = torch.full((4,), 1e-3, dtype=torch.float64)
    got = torch.tensor([1.0, float("nan"), 1.0, 1.0])
    assert math.isinf(R.max_ratio(got, ref, bound))
    assert not R.within(got, ref, bound)
