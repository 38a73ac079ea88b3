"""The corr-block protocol on the GPU (SURVEY.md section 8(b) row 2; ptlflow/models/raft/corr.py:104-118):
``get_corr_block(fmap1, fmap2, num_levels, radius, alternate_corr)`` built from the reference's NCHW tensors, called with
``coords [B,2,H,W]``, returning ``[B, L*(2r+1)^2, H, W]`` contiguous in coords' dtype -- against the vectors the
reference's own CorrBlock / IterativeCorrBlock wrote (tests/golden/op_corr_lookup.npz, op_alt_corr.npz).
This is the seam the sibling ``corr.py`` copies bind to (appendix E): also exercised here are the single-level r = 4
lookup of the FlowFormer decoder (flowformer/decoder.py:262-280) and SEA-RAFT's per-level volumes against a separately
sized target grid (sea_raft/corr.py:77-83)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden
from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _fmaps(recipe):
    b, c, h, w = recipe["b"], recipe["c"], recipe["h"], recipe["w"]
    f1 = torch.from_numpy(synth.synth_normal("ops/fmap1", (b, c, h, w), recipe["seed"]))
    f2 = torch.from_numpy(synth.synth_normal("ops/fmap2", (b, c, h, w), recipe["seed"]))
    return f1, f2


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-5), (torch.float16, 4e-2)])
@pytest.mark.parametrize("memory_format", [torch.contiguous_format, torch.channels_last])
def test_corr_block_against_reference_vectors(dtype, tol, memory_format):
    from ptlflow_b200.models.raft.corr import CorrBlock, get_corr_block

    recipe, g = load_golden("op_corr_lookup")
    f1, f2 = _fmaps(recipe)
    f1 = f1.to(DEV, dtype).contiguous(memory_format=memory_format)
    f2 = f2.to(DEV, dtype).contiguous(memory_format=memory_format)
    corr_fn = get_corr_block(f1, f2, num_levels=recipe["levels"], radius=recipe["radius"], alternate_corr=False)
    assert isinstance(corr_fn, CorrBlock)
    coords = torch.from_numpy(g["coords"]).to(DEV, dtype)  # the reference hands coords in the model dtype (raft.py:106)
    out = corr_fn(coords)
    assert out.shape == g["lookup"].shape and out.dtype == dtype and out.is_contiguous()
    # f16 coordinates are quantised by the CALLER here (0.03-0.06 px at x ~ 100): compare with the oracle at the same coords
    ref = O.corr_lookup(O.corr_pyramid(O.corr_volume(*_fmaps(recipe)), recipe["levels"]), coords.float().cpu(), recipe["radius"])
    assert (out.float().cpu() - ref).abs().max().item() < tol
    if dtype == torch.float32:
        assert np.abs(out.cpu().numpy() - g["lookup"]).max() < tol
    out2 = corr_fn(coords + 0.5)  # constructed once, called `iters` times
    assert (out2 - out).abs().max().item() > 0


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-5), (torch.float16, 4e-2)])
def test_alternate_corr_block_against_reference_vectors(dtype, tol):
    from ptlflow_b200.models.raft.corr import AlternateCorrBlock, get_corr_block

    recipe, g = load_golden("op_alt_corr")
    f1, f2 = _fmaps(recipe)
    corr_fn = get_corr_block(f1.to(DEV, dtype), f2.to(DEV, dtype), num_levels=recipe["levels"], radius=recipe["radius"], alternate_corr=True)
    assert isinstance(corr_fn, AlternateCorrBlock)
    coords = torch.from_numpy(g["coords"]).to(DEV, dtype)
    out = corr_fn(coords)
    assert out.shape == g["lookup"].shape and out.dtype == dtype
    ref = O.alt_corr_lookup(f1, f2, coords.float().cpu(), recipe["radius"], recipe["levels"])
    assert (out.float().cpu() - ref).abs().max().item() < tol
    if dtype == torch.float32:
        assert np.abs(out.cpu().numpy() - g["lookup"]).max() < tol


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-5), (torch.bfloat16, 2e-1)])
def test_flowformer_single_level_lookup(dtype, tol):
    """FlowFormer's encode_flow_token (decoder.py:262-280): ONE level, r = 4, cost maps WITHOUT the 1/sqrt(C) scale
    (encoder.py:543-561) -- the same kernels with levels = 1 and scale = 1."""
    from ptlflow_b200 import ops

    b, c, h, w = 1, 64, 27, 40  # odd sizes: no tensor-core tile divides them
    f1 = torch.from_numpy(synth.synth_normal("ff/f1", (b, c, h, w), 3))
    f2 = torch.from_numpy(synth.synth_normal("ff/f2", (b, c, h, w), 3))
    coords = O.coords_grid(b, h, w) + torch.from_numpy(synth.synth_normal("ff/c", (b, 2, h, w), 3, scale=6.0))
    pm = lambda t: t.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)  # noqa: E731
    (cost,) = ops.corr_volume_build_ex(pm(f1), pm(f2), levels=1, scale=1.0)
    assert cost.shape == (b * h * w, h, w)
    look = ops.corr_lookup([cost], coords.permute(0, 2, 3, 1).contiguous().to(DEV), 4, (h, w), nchw=True, out_dtype=torch.float32)
    vol = O.corr_volume(f1, f2) * (c ** 0.5)
    ref = O.corr_lookup([vol], coords, 4)
    assert look.shape == (b, 81, h, w)
    assert (look.cpu() - ref).abs().max().item() < tol * (c ** 0.5)


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-5), (torch.float16, 4e-2)])
def test_sea_raft_pyramid_of_volumes(dtype, tol):
    """SEA-RAFT style pyramid (sea_raft/corr.py:77-83): one all-pairs product PER LEVEL of the full-resolution fmap1 against
    fmap2 halved by bilinear interpolation (align_corners=False), instead of average-pooling the volume; same lookup."""
    from ptlflow_b200 import ops

    b, c, h, w = 2, 128, 24, 40
    f1 = torch.from_numpy(synth.synth_normal("sea/f1", (b, c, h, w), 4))
    f2 = torch.from_numpy(synth.synth_normal("sea/f2", (b, c, h, w), 4))
    coords = O.coords_grid(b, h, w) + torch.from_numpy(synth.synth_normal("sea/c", (b, 2, h, w), 4, scale=4.0))
    pm = lambda t: t.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)  # noqa: E731
    pyr, ref_pyr, t2 = [], [], f2
    for lvl in range(3):
        (v,) = ops.corr_volume_build_ex(pm(f1), pm(t2), levels=1, scale=c ** -0.5)  # targets_hw = t2's own grid
        assert v.shape == (b * h * w, t2.shape[-2], t2.shape[-1])
        pyr.append(v)
        a = f1.reshape(b, c, h * w).transpose(1, 2)
        ref_pyr.append((torch.bmm(a, t2.reshape(b, c, -1)) * c ** -0.5).reshape(b * h * w, 1, t2.shape[-2], t2.shape[-1]))
        t2 = F.interpolate(t2, scale_factor=0.5, mode="bilinear", align_corners=False)
    for v, r in zip(pyr, ref_pyr):
        assert (v.float().cpu() - r[:, 0]).abs().max().item() < tol
    look = ops.corr_lookup(pyr, coords.permute(0, 2, 3, 1).contiguous().to(DEV), 4, (h, w), nchw=True, out_dtype=torch.float32,
                           level_hw=[tuple(p.shape[-2:]) for p in pyr])
    ref = O.corr_lookup(ref_pyr, coords, 4)
    assert (look.cpu() - ref).abs().max().item() < 2 * tol


# ------------------------------------------------------------------------------------------
# tiled pyramid (64-byte tiles): what the refinement loop uses for f16 / bf16
# ------------------------------------------------------------------------------------------
TILED_CASES = [
    # b, c, h, w, levels, radius, dtype, tol
    (2, 256, 24, 40, 4, 4, torch.float16, 2e-2),
    (1, 256, 55, 128, 4, 4, torch.float16, 2e-2),   # the config-2 grid: odd height, 2 x 2 tile patches exactly
    (1, 128, 27, 45, 4, 4, torch.float16, 2e-2),    # odd everything: partial tiles, pad columns, floor-dropped rows / columns
    (1, 64, 9, 17, 3, 3, torch.float16, 2e-2),      # a grid smaller than one patch pair per row; radius 3 / 3 levels (raft_small-like)
    (1, 256, 16, 24, 1, 4, torch.bfloat16, 1.5e-1), # single level (FlowFormer)
    (3, 192, 13, 33, 2, 4, torch.bfloat16, 1.5e-1),
]


@pytest.mark.parametrize("b,c,h,w,levels,radius,dtype,tol", TILED_CASES)
def test_tiled_volume_and_lookup(b, c, h, w, levels, radius, dtype, tol):
    from ptlflow_b200 import ops

    f1 = torch.from_numpy(synth.synth_normal("tl/f1", (b, c, h, w), 11))
    f2 = torch.from_numpy(synth.synth_normal("tl/f2", (b, c, h, w), 11))
    coords = O.coords_grid(b, h, w) + torch.from_numpy(synth.synth_normal("tl/c", (b, 2, h, w), 11, scale=6.0))
    coords[0, :, 0, 0] = torch.tensor([-40.0, -40.0])        # far out of bounds
    coords[0, :, 0, 1] = torch.tensor([float(w) - 0.5, float(h) - 0.5])  # straddles the bottom-right corner
    coords[0, :, 0, 2] = torch.tensor([0.0, 0.0])            # integer coordinates: zero fractional weights
    coords[0, :, 1, 0] = torch.tensor([7.0, 3.25])           # window starts at tile column offset 7 -> third chunk
    pm = lambda t: t.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)  # noqa: E731
    pyr = ops.corr_volume_build_tiled(pm(f1), pm(f2), levels)
    # storage rounding of the features is part of the operator's contract: the oracle sees the rounded features
    f1r, f2r = f1.to(dtype).float(), f2.to(dtype).float()
    ref_pyr = O.corr_pyramid(O.corr_volume(f1r, f2r), levels)
    for l, (p, r) in enumerate(zip(pyr, ref_pyr)):
        dense = ops.untile_level(p, h >> l, w >> l)
        assert dense.shape == r[:, 0].shape
        err = (dense.float().cpu() - r[:, 0]).abs().max().item()
        assert err < tol, f"level {l}: {err}"
    look = ops.corr_lookup_tiled(pyr, coords.permute(0, 2, 3, 1).contiguous().to(DEV), radius, (h, w))
    planes = levels * (2 * radius + 1) ** 2
    assert look.shape == (b, h, w, (planes + 7) // 8 * 8)
    ref = O.corr_lookup(ref_pyr, coords, radius)
    got = look[..., :planes].permute(0, 3, 1, 2).float().cpu()
    assert (got - ref).abs().max().item() < 2 * tol
    assert look[..., planes:].abs().max().item() == 0
    # the tiled lookup reads exactly what the dense lookup reads from the same (stored) values
    dense_pyr = [ops.untile_level(p, h >> l, w >> l) for l, p in enumerate(pyr)]
    look_d = ops.corr_lookup(dense_pyr, coords.permute(0, 2, 3, 1).contiguous().to(DEV), radius, (h, w), nchw=True, out_dtype=torch.float32)
    assert (got - look_d.cpu()).abs().max().item() < (2e-3 if dtype == torch.float16 else 1.6e-2) * max(1.0, ref.abs().max().item())


def test_tiled_lookup_pad_columns_are_masked():
    """Pad columns / rows of the tiled maps may hold anything: poison them and look up again."""
    from ptlflow_b200 import ops

    b, c, h, w, levels, radius = 1, 64, 10, 13, 2, 4
    f1 = torch.from_numpy(synth.synth_normal("tp/f1", (b, c, h, w), 12))
    f2 = torch.from_numpy(synth.synth_normal("tp/f2", (b, c, h, w), 12))
    coords = (O.coords_grid(b, h, w) + torch.from_numpy(synth.synth_normal("tp/c", (b, 2, h, w), 12, scale=3.0))).permute(0, 2, 3, 1).contiguous().to(DEV)
    pm = lambda t: t.permute(0, 2, 3, 1).contiguous().to(DEV, torch.float16)  # noqa: E731
    pyr = ops.corr_volume_build_tiled(pm(f1), pm(f2), levels)
    a = ops.corr_lookup_tiled(pyr, coords, radius, (h, w)).clone()
    for l, p in enumerate(pyr):
        hl, wl = h >> l, w >> l
        ty, tx = (hl + 3) // 4, (wl + 7) // 8
        v = p.view(p.shape[0], ty, tx, 4, 8)
        ys = (torch.arange(ty, device=DEV)[:, None] * 4 + torch.arange(4, device=DEV)[None, :])[None, :, None, :, None]
        xs = (torch.arange(tx, device=DEV)[:, None] * 8 + torch.arange(8, device=DEV)[None, :])[None, None, :, None, :]
        v[((ys >= hl) | (xs >= wl)).expand_as(v)] = 1000.0
    bb = ops.corr_lookup_tiled(pyr, coords, radius, (h, w))
    assert torch.equal(a, bb)


# ------------------------------------------------------------------------------------------
# a4 on the tensor cores
# ------------------------------------------------------------------------------------------
OTF_CASES = [
    # b, c, h, w, levels, sigma (px of coordinate noise: small = smooth flow, large = rough -> SIMT pass), dtype, tol
    (1, 256, 24, 48, 4, 0.7, torch.float16, 2e-2),
    (2, 256, 27, 45, 4, 1.5, torch.float16, 2e-2),   # partial tiles on both axes, odd level sizes
    (1, 128, 16, 32, 3, 12.0, torch.float16, 2e-2),  # rough flow: most queries are flagged and recomputed
    (1, 256, 55, 128, 4, 2.0, torch.bfloat16, 1.5e-1),
    (1, 64, 9, 17, 2, 1.0, torch.float16, 2e-2),     # C = 64: a single K chunk
    (1, 128, 135, 240, 4, 1.0, torch.float16, 2e-2), # 1020 work items on 132 CTAs: every ring / region slot wraps several times
]


@pytest.mark.parametrize("b,c,h,w,levels,sigma,dtype,tol", OTF_CASES)
def test_onthefly_tensor_core(b, c, h, w, levels, sigma, dtype, tol):
    from ptlflow_b200 import ops

    f1 = torch.from_numpy(synth.synth_normal("otc/f1", (b, c, h, w), 31))
    f2 = torch.from_numpy(synth.synth_normal("otc/f2", (b, c, h, w), 31))
    smooth = torch.from_numpy(synth.synth_normal("otc/s", (b, 2, 1, 1), 31, scale=3.0))  # a common displacement per sample
    coords = O.coords_grid(b, h, w) + smooth + torch.from_numpy(synth.synth_normal("otc/c", (b, 2, h, w), 31, scale=sigma))
    coords[0, :, 0, 0] = torch.tensor([-60.0, -60.0])                 # far out of bounds: zero window
    coords[0, :, 0, 1] = torch.tensor([float(w) + 2.5, float(h) - 1.25])  # straddles the right / bottom border
    coords[0, :, 1, 0] = torch.tensor([float("nan"), 0.0])            # non-finite: zero window like the SIMT kernel
    pm = lambda t: t.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)  # noqa: E731
    cpm = coords.permute(0, 2, 3, 1).contiguous().to(DEV)
    pyr = ops.feature_pyramid(pm(f2), levels)
    out = ops.corr_lookup_onthefly_tc(pm(f1), pyr, cpm, 4)
    planes = levels * 81
    simt = ops.corr_lookup_onthefly(pm(f1), pyr, cpm, 4, nchw=False, out_stride=out.shape[-1])
    flagged = int(out._pfb_flags.sum().item())
    d = (out[..., :planes].float() - simt[..., :planes].float()).abs().max().item()
    scale = max(1.0, simt[..., :planes].float().abs().max().item())
    assert d < tol * scale, f"tensor-core vs SIMT on-the-fly: {d} (flagged {flagged} of {b * h * w})"
    assert out[..., planes:].abs().max().item() == 0
    if sigma < 3:
        assert flagged < 0.2 * b * h * w, f"smooth flow but {flagged} of {b * h * w} queries left the tile regions"
    # and against the oracle (features rounded to the storage type first, as the operator's contract says)
    coords_ref = torch.nan_to_num(coords, nan=-1e6)
    ref = O.alt_corr_lookup(f1.to(dtype).float(), f2.to(dtype).float(), coords_ref, 4, levels)
    got = out[..., :planes].permute(0, 3, 1, 2).float().cpu()
    assert (got - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())
