"""GPU: CRAFT's a23 kernels against float64 with per-element bounds, the volume's statistics bit-identical across runs and under graph
replay, the fp32 fixtures eagerly and replayed, and the half-precision flow against the fp32 model at 436 x 1024."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import craft_oracle as CR  # noqa: E402
from helpers import DEV, DTYPES, U, _model, case_recipe, check_fp32_fixture, check_half_against_fp32  # noqa: E402

pytestmark = pytest.mark.gpu


def _bias(R, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(2 * R + 1, 2 * R + 1, generator=g, dtype=torch.float64)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H, W, R, mask, scale", [(5, 7, 2, -1, 1.0), (9, 11, 7, 3, 1.0), (6, 8, 0, -1, 40.0), (17, 17, 15, -1, 40.0)])
def test_window_softmax_against_float64(dtype, H, W, R, mask, scale):
    """Clamp (scale 40 pushes logits past 100), window bias, mask radius and the row softmax; bound: the logits' storage rounding
    (|x| u, through the softmax at most 2 |x| u p relative) plus the output's rounding."""
    from ptlflow_b200 import ops

    M, B, N = 2, 2, H * W
    g = torch.Generator().manual_seed(H * 31 + R)
    x = (torch.randn(M * B * N, N, generator=g, dtype=torch.float64) * scale).to(dtype)
    bias = _bias(R, R) * 0.5
    x64 = x.double()
    s = x64.clamp(-100, 100) if x64.max() > 100 else x64
    s = s.view(M, B, N, N) + CR.window_bias(bias, H, W).double()
    if mask > 0:
        s = s + CR.chebyshev_mask(H, W, mask).double()
    ref = torch.softmax(s, -1).view(M * B * N, N)
    xd = x.to(DEV)
    got = ops.craft_window_softmax(xd, H, W, bias.float().reshape(-1).contiguous().to(DEV), R, ops.craft_clamp_flag(xd), mask).double().cpu()
    u = max(U[dtype], 2.0 ** -23)
    bound = ref * (4 * 100 * 2.0 ** -23 + 2 * u) + 1e-7
    assert ((got - ref).abs() <= bound).all(), (got - ref).abs().max().item()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M, F_", [(1, 128), (4, 128), (2, 256), (4, 256)])
def test_mode_aggregate_against_float64(dtype, M, F_):
    from ptlflow_b200 import ops

    P = 301
    g = torch.Generator().manual_seed(M * F_)
    feat = torch.randn(P, M * F_, generator=g, dtype=torch.float64).to(dtype)
    skip = torch.randn(P, F_, generator=g, dtype=torch.float64).to(dtype)
    w = torch.randn(F_, generator=g, dtype=torch.float64) * 0.3
    coeff = 0.8
    y = feat.double().view(P, M, F_)
    pi = torch.softmax(y @ w, dim=1)
    t = coeff * skip.double() + (pi[..., None] * y).sum(1)
    ref = torch.nn.functional.layer_norm(t, (F_,), eps=1e-12)
    got = ops.craft_mode_aggregate(feat.to(DEV), M, w.float().to(DEV), coeff, skip.to(DEV)).double().cpu()
    tol = 2e-5 if dtype == torch.float32 else 4 * U[dtype] * (1 + ref.abs())
    assert ((got - ref).abs() <= tol).all(), (got - ref).abs().max().item()


def _volume_case(dtype, M, B, H, W, R, scale, seed):
    g = torch.Generator().manual_seed(seed)
    N = H * W
    scores = (torch.randn(M * B * N, N, generator=g, dtype=torch.float64) * scale).to(dtype)
    bias = _bias(R, seed)
    a = 0.6
    s = scores.double()
    s = (s.clamp(-100, 100) if s.max() > 100 else s).view(M, B, N, N) + 0.5 * CR.window_bias(bias, H, W).double()
    mix = s[0] if M == 1 else (torch.softmax(a * s, 0) * s).sum(0)
    ref = torch.nn.functional.layer_norm(mix.reshape(B, -1), (N * N,), eps=1e-12).reshape(B * N, H, W)
    return scores, (0.5 * bias).float().reshape(-1).contiguous(), a, ref


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M, B, H, W, R, scale", [(4, 1, 7, 9, 7, 1.0), (2, 2, 13, 11, 3, 30.0), (1, 2, 5, 6, 0, 1.0)])
def test_volume_norm_against_float64(dtype, M, B, H, W, R, scale):
    """Level 0 of the inter-frame volume: the fp32 mix of the stored scores, normalised with fp64 statistics; bound: the mix's fp32
    error relative to the sample's standard deviation plus the level's storage rounding."""
    from ptlflow_b200 import ops

    scores, bias, a, ref = _volume_case(dtype, M, B, H, W, R, scale, H * W + M)
    sd = scores.to(DEV)
    got = ops.craft_volume_norm(sd, M, B, H, W, a, bias.to(DEV), R, ops.craft_clamp_flag(sd)).double().cpu()
    tol = 1e-4 if dtype == torch.float32 else 2 * U[dtype] * ref.abs() + 1e-4
    assert ((got - ref).abs() <= tol).all(), (got - ref).abs().max().item()


def test_volume_statistics_are_bit_identical_on_replay():
    from ptlflow_b200 import ops

    scores, bias, a, _ = _volume_case(torch.bfloat16, 4, 2, 20, 24, 7, 10.0, 7)
    sd, bd = scores.to(DEV), bias.to(DEV)
    run = lambda: ops.craft_volume_norm(sd, 4, 2, 20, 24, a, bd, 7, ops.craft_clamp_flag(sd))  # noqa: E731
    first, second = run(), run()
    assert torch.equal(first, second)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = run()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first)


@pytest.mark.parametrize("name", CR.E2E)
def test_craft_fp32_fixtures(name):
    rec = case_recipe(CR, name)
    sd, img, kw = CR.e2e_inputs(rec)
    check_fp32_fixture(_model("craft", sd, **kw), img, name, 1e-4)


HALF_GATES = {torch.float16: (8e-2, 2e-2), torch.bfloat16: (5e-1, 1e-1)}


def test_half_precision_against_fp32_436x1024():
    rec = dict(case_recipe(CR, "e2e_craft_default"), batch=1, height=436, width=1024)
    sd, img, _ = CR.e2e_inputs(rec)
    check_half_against_fp32(lambda dtype: _model("craft", sd, dtype, iters=12), img.to(DEV), HALF_GATES, "craft at 436x1024, 12 iterations")


def _fused_case(dtype, M, B, H, W, R, scale, seed):
    """q1 / k2 [B,H,W,256] in the storage type and the float64 level 0 [B*N, H, W] of the fused volume they give."""
    g = torch.Generator().manual_seed(seed)
    N, d = H * W, 256 // M
    q1 = (torch.randn(B, H, W, 256, generator=g, dtype=torch.float64) * scale).to(dtype)
    k2 = (torch.randn(B, H, W, 256, generator=g, dtype=torch.float64) * scale).to(dtype)
    bias = 0.5 * _bias(R, seed)
    a = 0.6
    q = q1.double().view(B, N, M, d).transpose(1, 2)
    k = k2.double().view(B, N, M, d).transpose(1, 2)
    s = q @ k.transpose(-1, -2) / d ** 0.5  # [B, M, N, N]
    flagged = s.max() > 100
    s = (s.clamp(-100, 100) if flagged else s) + CR.window_bias(bias, H, W).double()
    mix = s[:, 0] if M == 1 else (torch.softmax(a * s, 1) * s).sum(1)
    ref = torch.nn.functional.layer_norm(mix.reshape(B, -1), (N * N,), eps=1e-12).reshape(B * N, H, W)
    return q1, k2, bias.float().reshape(-1).contiguous(), a, ref, mix.reshape(B, -1).std(1).min().item(), s.abs().max().item()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M, B, H, W, R, scale", [(4, 1, 8, 8, 7, 1.0), (2, 2, 17, 17, 3, 1.0), (1, 1, 9, 20, 0, 1.0), (4, 2, 13, 23, 15, 5.0)])
def test_fused_volume_against_float64_and_the_fallback(dtype, M, B, H, W, R, scale):
    """pfb_craft_volume_tiled on ragged grids (patches and query blocks cut by the map, one case past the clip): every level against
    float64 (bound: fp32 mix and statistics, then the storage rounding of the stored value), and level 0 against the materialised route
    built from the same operands (which also rounds the per-mode scores to the storage type)."""
    from ptlflow_b200 import ops

    q1, k2, bias, a, ref, std, smax = _fused_case(dtype, M, B, H, W, R, scale, H * W + M)
    bd = bias.to(DEV)
    pyr = ops.craft_volume_tiled(q1.to(DEV).contiguous(), k2.to(DEV).contiguous(), M, a, bd, R, 4)
    ref_pyr = CR.O.corr_pyramid(ref[:, None], 4)
    u = U[dtype]
    for l in range(4):
        got = ops.untile_level(pyr[l], H >> l, W >> l).double().cpu()
        r = ref_pyr[l][:, 0]
        assert got.shape == r.shape
        bound = 2 * u * r.abs() + 2e-4 * (1 + smax / std)
        assert ((got - r).abs() <= bound).all(), (l, (got - r).abs().max().item())
    N, d = H * W, 256 // M
    qh = q1.to(DEV).view(B, N, M, d).permute(2, 0, 1, 3).contiguous().view(M * B, H, W, d)
    kh = k2.to(DEV).view(B, N, M, d).permute(2, 0, 1, 3).contiguous().view(M * B, H, W, d)
    scores = ops.corr_volume_build_ex(qh, kh, 1, scale=d ** -0.5)[0].view(M * B * N, N)
    dense = ops.craft_volume_norm(scores, M, B, H, W, a, bd, R, ops.craft_clamp_flag(scores)).double().cpu()
    fused0 = ops.untile_level(pyr[0], H, W).double().cpu()
    assert ((fused0 - dense).abs() <= 4 * u * (ref.abs() + smax / std) + 1e-3).all(), (fused0 - dense).abs().max().item()


def test_fused_volume_is_bit_identical_on_replay():
    """Every in-map value of every level (the pad cells of a level's last tiles are not part of the volume: the lookup masks them)."""
    from ptlflow_b200 import ops

    q1, k2, bias, a, _, _, _ = _fused_case(torch.bfloat16, 4, 2, 20, 24, 7, 1.0, 9)
    q1, k2, bd = q1.to(DEV).contiguous(), k2.to(DEV).contiguous(), bias.to(DEV)
    def run():
        pyr = ops.craft_volume_tiled(q1, k2, 4, a, bd, 7, 4)
        return [ops.untile_level(p, 20 >> l, 24 >> l) for l, p in enumerate(pyr)]

    first, second = run(), run()
    assert all(torch.equal(x, y) for x, y in zip(first, second))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = run()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(out, first))


def test_model_selects_the_fused_volume_by_dtype():
    """f16 / bf16 with the default (radius, levels) and 64-channel modes take the tiled pyramid; fp32 the dense one."""
    rec = case_recipe(CR, "e2e_craft_default")
    sd, img, kw = CR.e2e_inputs(rec)
    for dtype, layout in ((torch.float32, 0), (torch.bfloat16, 1)):
        m = _model("craft", sd, dtype, **kw)
        fmap = torch.zeros(1, 16, 20, 256, dtype=dtype, device=DEV)
        eng = m._get_engine(dtype, torch.device(DEV))
        assert eng.craft_volume(fmap, fmap)[1] == layout
