"""The float64 references and per-element bounds of the normalisation passes and the two first convolutions
(norm_reference.py) on the CPU: each reference rounded once to the storage type passes, and each of a set of plausible kernel
bugs, planted into the float64 result at a shape the GPU conformance tests run, is rejected, in f16 and in bf16 -- by the bound,
or for the counting faults the bound is too loose to see, by the exact-sum check on dyadic inputs."""
import pytest
import torch
import torch.nn.functional as F

import conv_reference as R
import norm_reference as N

DTYPES = [torch.float16, torch.bfloat16]
IDS = ["f16", "bf16"]
EPS = 1e-5


def _stats(x, unbiased=False):
    """Exact per-(image, channel) mean and variance of x [B,H,W,C] as [B,1,1,C]."""
    x = x.double()
    mean = x.mean(dim=(1, 2), keepdim=True)
    var = x.var(dim=(1, 2), keepdim=True, unbiased=unbiased)
    return mean, var


def _group_stats(x, bias, group):
    B, H, W, C = x.shape
    v = (x.double() + bias).view(B, H, W, C // group, group)
    mean = v.mean(dim=(1, 2, 4), keepdim=True)
    var = v.var(dim=(1, 2, 4), keepdim=True, unbiased=False)
    rs = lambda t: t.expand(B, 1, 1, C // group, group).reshape(B, 1, 1, C)  # noqa: E731
    return rs(mean), rs(var)


def _rejected(got, ref, bound, dtype):
    assert R.within(R.q(ref, dtype), ref, bound), "the rounded reference must pass"
    return not R.within(R.q(got, dtype), ref, bound)


# ---- instance norm -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_instance_norm_eps_outside_sqrt_rejected(dtype):
    x = N.norm_input(3, 31, 33, 24, dtype, 1).double()
    ref, bound = N.instance_norm(x, dtype)
    mean, var = _stats(x)
    assert _rejected((x - mean) / (var.sqrt() + EPS), ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_instance_norm_unbiased_variance_rejected(dtype):
    x = N.norm_input(3, 1, 7, 64, dtype, 2).double()
    ref, bound = N.instance_norm(x, dtype)
    mean, var = _stats(x, unbiased=True)
    assert _rejected((x - mean) / (var + EPS).sqrt(), ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_instance_norm_reversed_image_stats_rejected(dtype):
    """The statistics kernel walks the images in descending order: image b normalised with the sums of image B-1-b."""
    x = N.norm_input(3, 31, 33, 24, dtype, 3).double()
    ref, bound = N.instance_norm(x, dtype, relu=True)
    mean, var = _stats(x)
    got = ((x - mean.flip(0)) / (var.flip(0) + EPS).sqrt()).clamp_min(0.0)
    assert _rejected(got, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_instance_norm_residual_without_outer_relu_rejected(dtype):
    x = N.norm_input(3, 31, 33, 64, dtype, 4).double()
    res = N.norm_input(3, 31, 33, 64, dtype, 5).double()
    ref, bound = N.instance_norm(x, dtype, relu=True, residual=res)
    mean, var = _stats(x)
    y = ((x - mean) / (var + EPS).sqrt()).clamp_min(0.0)
    assert _rejected(res + y, ref, bound, dtype)


# ---- group norm ----------------------------------------------------------------------------------------------------------
def _gn_operands(dtype, C=64, group=16):
    x = N.norm_input(3, 31, 33, C, dtype, 6).double()
    g = torch.Generator().manual_seed(7)
    bias = torch.randn(C, generator=g, dtype=torch.float64).float().double()
    gamma = (1.0 + 0.5 * torch.randn(C, generator=g, dtype=torch.float64)).float().double()
    beta = (0.3 * torch.randn(C, generator=g, dtype=torch.float64)).float().double()
    ref, bound = N.group_norm(x, dtype, group, bias=bias, gamma=gamma, beta=beta, relu=True)
    return x, bias, gamma, beta, group, ref, bound


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_group_norm_bias_in_mean_only_rejected(dtype):
    """The bias folded into the group's sum but not into its sum of squares."""
    x, bias, gamma, beta, group, ref, bound = _gn_operands(dtype)
    B, H, W, C = x.shape
    mean, _ = _group_stats(x, bias, group)
    q = (x * x).view(B, H, W, C // group, group).mean(dim=(1, 2, 4), keepdim=True)
    q = q.expand(B, 1, 1, C // group, group).reshape(B, 1, 1, C)
    var = (q - mean * mean).clamp_min(0.0)
    got = ((x + bias - mean) / (var + EPS).sqrt() * gamma + beta).clamp_min(0.0)
    assert _rejected(got, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_group_norm_bias_not_folded_rejected(dtype):
    """The statistics of x alone (the bias still in the shift)."""
    x, bias, gamma, beta, group, ref, bound = _gn_operands(dtype)
    mean, var = _group_stats(x, torch.zeros_like(bias), group)
    got = ((x + bias - mean) / (var + EPS).sqrt() * gamma + beta).clamp_min(0.0)
    assert _rejected(got, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_group_norm_affine_of_first_channel_rejected(dtype):
    x, bias, gamma, beta, group, ref, bound = _gn_operands(dtype)
    first = torch.arange(x.shape[-1]) // group * group
    mean, var = _group_stats(x, bias, group)
    got = ((x + bias - mean) / (var + EPS).sqrt() * gamma[first] + beta[first]).clamp_min(0.0)
    assert _rejected(got, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES + [torch.float32], ids=IDS + ["f32"])
def test_rounded_references_pass(dtype):
    """Every mode of the three passes, on realistic and dyadic inputs, rounded once to the storage type."""
    for exact in (False, True):
        x = N.norm_input(3, 31, 33, 24, dtype, 8, exact=exact).double()
        res = N.norm_input(3, 31, 33, 24, dtype, 9, exact=exact).double()
        bias = torch.linspace(-2.0, 2.0, 24, dtype=torch.float64)
        cases = [N.instance_norm(x, dtype, relu=relu, residual=r) for relu in (False, True) for r in (None, res)]
        cases += [N.group_norm(x, dtype, 8, bias=bias, gamma=bias.flip(0), beta=0.5 * bias, relu=True, residual=res),
                  N.group_norm(x, dtype, 8, relu=False),
                  N.bias_act(x, bias, dtype, relu=True, residual=res), N.bias_act(x, None, dtype)]
        for ref, bound in cases:
            assert R.within(R.q(ref, dtype), ref, bound)


# ---- exact sums ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
@pytest.mark.parametrize("fault", ["pixel_dropped", "pixel_counted_twice", "image_swapped"])
def test_exact_sums_reject_counting_faults(fault, dtype):
    """On dyadic inputs the workspace sums must equal the float64 sums: one dropped or double-counted pixel shows, however
    small it is against the sum."""
    x = N.norm_input(3, 64, 128, 64, dtype, 10, exact=True).double()
    s, q = N.sums(x)
    ws = torch.stack([s, q], -1)
    N.assert_sums_equal(ws, s, q)
    bad = ws.clone()
    if fault == "pixel_dropped":
        bad[1, 5] -= torch.stack([x[1, 63, 127, 5], x[1, 63, 127, 5] ** 2])
    elif fault == "pixel_counted_twice":
        bad[2, 40] += torch.stack([x[2, 0, 64, 40], x[2, 0, 64, 40] ** 2])
    else:
        bad = bad.flip(0)
    with pytest.raises(AssertionError):
        N.assert_sums_equal(bad, s, q)


def test_stats_k_follows_the_launch():
    # C = 64: 8 octets, 32 lanes, a 2-level shuffle tree, 8 warps; C = 24: 3 octets, 85 lanes, no tree; C = 512: 4 lanes
    assert N.stats_k(220 * 512, 64) == 48 + 2 + 8 + 1
    assert N.stats_k(1023, 24) == 1 + 0 + 85 + 1
    assert N.stats_k(8192, 512) == 192 + 0 + 4 + 1
    assert N.stats_k(1, 8) == 1 + 5 + 8 + 1
    assert N.first_conv_items(16, 220, 512, 132) == (16 * 110 * 4, 54)
    assert N.first_conv_items(13, 21, 100, 132) == (143, 2)


# ---- first convolution (7x7, stride 2) -------------------------------------------------------------------------------------
def _conv1(dtype, N_=2, H=20, W=258, seed=11):
    x = N.frames(N_, H, W, dtype, seed)[..., :3].double()
    g = torch.Generator().manual_seed(seed + 1)
    w = R.q(0.12 * torch.randn((64, 3, 7, 7), generator=g, dtype=torch.float64), dtype)
    ref, bound, acc, E, n = N.first_conv(x, w, None, dtype, relu=False)
    return x, w, ref, bound, acc


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_first_conv_top_row_skipped_rejected(dtype):
    x, w, ref, bound, acc = _conv1(dtype)
    top = torch.zeros_like(x)
    top[:, 0] = x[:, 0]
    contrib, _, _ = R.conv_terms([top], w, stride=2)
    assert _rejected(acc - contrib, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_first_conv_window_shifted_at_segment_edge_rejected(dtype):
    """Output pixel 127, the last of the first 128-pixel segment, reads its window one input pixel to the right."""
    x, w, ref, bound, acc = _conv1(dtype)
    shifted = torch.zeros_like(x)
    shifted[:, :, :-1] = x[:, :, 1:]
    moved, _, _ = R.conv_terms([shifted], w, stride=2)
    got = acc.clone()
    got[:, :, 127] = moved[:, :, 127]
    assert _rejected(got, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_first_conv_second_row_phase_misplaced_rejected(dtype):
    """The second row phase (odd output rows) written one pair further down."""
    x, w, ref, bound, acc = _conv1(dtype)
    got = acc.clone()
    got[:, 3::2] = acc[:, 1:-2:2]
    assert _rejected(got, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_first_conv_sum_bound_holds_for_rounded_accumulators(dtype):
    """The statistics bound covers sums of the accumulator values rounded anywhere inside E (here: to the storage type, which
    is coarser than the accumulator)."""
    x, w, ref, bound, acc = _conv1(dtype)
    _, _, acc, E, _ = N.first_conv(x, w, None, dtype, relu=False)
    v = R.q(acc, dtype)
    assert ((v - acc).abs() <= E + R.RHO[dtype] * acc.abs()).all()
    n_items, per_cta = N.first_conv_items(2, 10, 129, 132)
    ds, dq = N.conv_sum_errors(acc, E + R.RHO[dtype] * acc.abs(), N.first_conv_k(per_cta))
    s, q = N.sums(acc)
    N.assert_sums_within(torch.stack(N.sums(v), -1), s, q, ds, dq)


# ---- convf1 ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_flow_conv_lo_half_dropped_rejected(dtype):
    """Dropping the lo half is within output rounding on a random flow; a smooth 100-400 px flow under zero-sum filters
    (the motion encoder's cancellation: the filters see differences of large values) exposes it."""
    flow = N.smooth_flow(1, 55, 128, 12)
    w = R.q(N.sparse_filter(128, 2, 6, 13, zero_sum=True), dtype)
    bias = R.q(0.3 * torch.randn(128, generator=torch.Generator().manual_seed(14), dtype=torch.float64), torch.float32)
    ref, bound = N.flow_conv(flow, w, bias, dtype)
    bad, _ = N.flow_conv(flow, w, bias, dtype, lo=False)
    assert _rejected(bad, ref, bound, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_flow_conv_references_pass(dtype):
    g = torch.Generator().manual_seed(15)
    bias = R.q(0.3 * torch.randn(128, generator=g, dtype=torch.float64), torch.float32)
    for flow, w in ((25.0 * torch.randn((2, 11, 21, 2), generator=g), 0.1 * torch.randn((128, 2, 7, 7), generator=g, dtype=torch.float64)),
                    (1e-4 * torch.randn((2, 11, 21, 2), generator=g), 0.1 * torch.randn((128, 2, 7, 7), generator=g, dtype=torch.float64)),
                    (N.smooth_flow(1, 9, 40, 16), N.sparse_filter(128, 2, 6, 17, zero_sum=True)),
                    (N.exact_flow(1, 9, 40, dtype, 18), N.sparse_filter(128, 2, 6, 19))):
        ref, bound = N.flow_conv(flow.float(), R.q(w, dtype), bias, dtype)
        assert R.within(R.q(ref, dtype), ref, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=IDS)
def test_exact_flow_splits_exactly(dtype):
    flow = N.exact_flow(2, 9, 40, dtype, 20)
    hi, lo = N.split_flow(flow, dtype)
    assert torch.equal(hi + lo, flow.double())
    assert lo.abs().max() > 0
    w = N.sparse_filter(128, 2, 6, 21, zero_sum=True)
    assert torch.equal(w.sum(dim=(2, 3)), torch.zeros(128, 2, dtype=torch.float64))
    assert w.abs().sum(dim=(1, 2, 3)).max() <= 3.0
    # the magnitude sum of every output stays below 2^7, the limit the exactness argument uses
    S = F.conv2d(flow.double().abs().permute(0, 3, 1, 2), w.abs(), padding=3)
    assert S.max() < 2.0 ** 7
