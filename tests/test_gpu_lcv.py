"""GPU: LCV -- the tiled lookup with explicit level sizes against the float64 lookup, the fp32 fixtures (eager and graph replay), LCV
with W = I against RAFT, the dense and tiled pyramids on a frozen grid, the f16 range of the learned layer, and half precision at
436x1024 against the fp32 model."""
import numpy as np
import pytest
import torch

import corr_reference as CR
import lcv_oracle as LO
from helpers import DEV, _model, case_recipe, check_fp32_fixture, check_half_against_fp32, load_golden
from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("radius,grid", [(4, (17, 21)), (4, (8, 8)), (3, (12, 16)), (3, (16, 20))])
def test_tiled_lookup_with_explicit_sizes_against_float64(dtype, radius, grid):
    from ptlflow_b200 import ops

    B, C_ = 2, 64
    H, W = grid
    levels = 4
    sizes, distinct = ops.corr_level_sizes(H, W, levels, 2 * radius + 1)
    g = torch.Generator(device=DEV).manual_seed(11)
    f1 = torch.randn(B, H, W, C_, device=DEV, generator=g).to(dtype)
    f2 = torch.randn(B, H, W, C_, device=DEV, generator=g).to(dtype)
    pyr = ops.corr_volume_build_tiled(f1, f2, distinct)
    pyr = pyr + [pyr[-1]] * (levels - distinct)  # the repeated levels are the same tensor
    coords = (O.coords_grid(B, H, W).to(DEV).permute(0, 2, 3, 1)
              + 3.0 * torch.randn(B, H, W, 2, device=DEV, generator=g)).contiguous()
    out = ops.corr_lookup_tiled(pyr, coords, radius, (H, W), level_hw=sizes)
    dense = [ops.untile_level(p, h, w).double() for p, (h, w) in zip(pyr, sizes)]
    ref, bound = CR.lookup(dense, coords.view(-1, 2), radius, dtype)
    planes = levels * (2 * radius + 1) ** 2
    got = out.view(B * H * W, -1)[:, :planes].double()
    assert (got - ref).abs().le(bound).all(), (got - ref).abs().max().item()
    assert not out.view(B * H * W, -1)[:, planes:].any()
    if distinct < levels:  # frozen levels really are read at coords / 2^l: level `distinct` differs from level `distinct - 1`
        K2 = (2 * radius + 1) ** 2
        a, b = got[:, (distinct - 1) * K2: distinct * K2], got[:, distinct * K2: (distinct + 1) * K2]
        assert (a - b).abs().max() > 0.1


@pytest.mark.parametrize("name", LO.E2E)
def test_fp32_fixtures_eager_and_replayed(name):
    rec = case_recipe(LO, name)
    sd, img, kw = LO.e2e_inputs(rec)
    check_fp32_fixture(_model(rec["model"], sd, **kw), img, name, 1e-4)


def _identity_form(sd, dim):
    sd = dict(sd)
    sd.update({"corr_block.raw_P": torch.eye(dim), "corr_block.raw_D": torch.zeros(dim), "corr_block.eye": torch.eye(dim)})
    return sd


@pytest.mark.parametrize("name,raft,dim", [("lcv_raft", "raft", 256), ("lcv_raft_small", "raft_small", 128)])
def test_identity_form_is_raft_where_every_level_pools(name, raft, dim):
    """W = I (the reference's initialisation): on a grid where every level pools LCV is RAFT (fed the frames with the channels
    reversed, as LCV keeps BGR); on a frozen grid it is not."""
    sd = synth.synth_state_dict(O.state_dict_shapes(raft), 21)
    lcv = _model(name, _identity_form(sd, dim), iters=4)
    ref = _model(raft, sd, iters=4)
    for (h, w), same in (((320, 384), True), ((128, 160), False)):
        img = torch.from_numpy(synth.synth_images(1, h, w, 22, "smooth")).to(DEV)
        with torch.no_grad():
            a = lcv({"images": img.flip(2)})["flows"]
            b = ref({"images": img})["flows"]
        err = (a - b).abs().max().item()
        print(f"{name} with W = I vs {raft} at {h}x{w}: max-abs {err:.2e} px")
        # W = I / sqrt(C) is exact, but the first convolution's reversed input channels reorder cuDNN's fp32 sums (measured on an H100:
        # 1.5e-5 px for lcv_raft, 5.8e-5 px for lcv_raft_small after 4 iterations)
        assert (err < 1e-4) if same else (err > 1e-3)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dense_and_tiled_pyramids_agree_on_a_frozen_grid(dtype, monkeypatch):
    from ptlflow_b200 import engine

    name = "e2e_lcv_raft_ragged"
    rec = case_recipe(LO, name)
    g = torch.from_numpy(load_golden(name)[1]["flows"])
    sd, img, kw = LO.e2e_inputs(rec)
    outs = {}
    for tiled in (True, False):
        monkeypatch.setattr(engine, "_TILED", tiled)
        m = _model("lcv_raft", sd, dtype, **kw)
        eng = m._get_engine(dtype, torch.device(DEV))
        f = torch.randn(1, 17, 21, 256, device=DEV).to(dtype)
        pyr, layout = eng.build_volume(f, f)
        assert layout == int(tiled) and len(pyr) == 4 and pyr[1] is pyr[2] is pyr[3] and pyr[0] is not pyr[1]
        with torch.no_grad():
            outs[tiled] = m({"images": img.to(DEV, dtype)})["flows_fp32"].float().cpu()
    tol = {torch.float16: 0.05, torch.bfloat16: 0.4}[dtype]
    for tiled, o in outs.items():
        e = (o - g).abs().max().item()
        print(f"lcv_raft {dtype} {'tiled' if tiled else 'dense'} vs the fp32 fixture: max-abs {e:.4f} px")
        assert e < tol
    assert (outs[True] - outs[False]).abs().max().item() < tol


# D = (1 + t) / (1 - t), t = atan(raw_D) 2 / pi: raw_D = 20.67 gives D = 64.0 on every channel, 63.66 gives D = 199.  With D = 199 the
# f16 volume overflows (measured max |<f1^T W / sqrt(C), f2>| 71168 on an H100, DESIGN.md section 5, LCV); f16 is checked at D = 64,
# the largest D an f16 engine takes without a warning, and bf16 at D = 199.
@pytest.mark.parametrize("dtype,raw_d", [(torch.float16, 20.67), (torch.bfloat16, 63.66)])
def test_learned_layer_range_with_a_large_diagonal(dtype, raw_d):
    """f1^T W / sqrt(C) in the storage type for a large D, on the fnet features of a real frame pair: the layer and the volume finite,
    and the layer within the storage type's rounding of the same layer in fp32 on the same features."""
    from ptlflow_b200 import ops

    sd = LO.synth_state_dict("lcv_raft", 31)
    sd["corr_block.raw_D"] = torch.full((256,), raw_d)
    img = torch.from_numpy(synth.synth_images(1, 436, 1024, 32, "smooth")).to(DEV)
    m32 = _model("lcv_raft", sd, torch.float32, iters=1)
    feats = m32.fnet.forward_pm(ops.preprocess_frames(img, (440, 1024), (2, 0), out_channels=4))
    f1 = feats[:1].to(dtype).contiguous()
    ref = ops.conv2d([f1.float()], m32._get_engine(torch.float32, torch.device(DEV)).learned, torch.empty_like(f1, dtype=torch.float32))
    mh = _model("lcv_raft", sd, dtype, iters=1)
    out = ops.conv2d([f1], mh._get_engine(dtype, torch.device(DEV)).learned, torch.empty_like(f1)).float()
    vol = ops.corr_volume_build_ex(out.to(dtype), feats[1:].to(dtype).contiguous(), 1, scale=1.0)[0].float()
    err = ((out - ref).abs() / ref.abs().max()).max().item()
    print(f"{dtype}: max |f1^T W / sqrt(C)| = {ref.abs().max().item():.1f} (max |f1| {f1.float().abs().max().item():.1f}), max |volume| "
          f"{vol.abs().max().item():.1f}; max-abs error / max {err:.2e}")
    assert torch.isfinite(out).all() and torch.isfinite(vol).all()
    assert err < {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}[dtype]


def test_f16_engine_warns_above_the_safe_diagonal():
    """An f16 engine whose learned D exceeds engine.LCV_F16_MAX_D warns when it is built; at D = 64 and in bf16 it does not."""
    import warnings

    from ptlflow_b200 import engine

    for dtype, raw_d, warns in ((torch.float16, 63.66, True), (torch.float16, 20.67, False), (torch.bfloat16, 63.66, False)):
        sd = LO.synth_state_dict("lcv_raft", 31)
        sd["corr_block.raw_D"] = torch.full((256,), raw_d)
        m = _model("lcv_raft", sd, dtype, iters=1)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            m._get_engine(dtype, torch.device(DEV))
        hit = [x for x in w if issubclass(x.category, RuntimeWarning) and "bfloat16" in str(x.message)]
        assert bool(hit) == warns, (dtype, raw_d, [str(x.message) for x in w])
    assert engine.LCV_F16_MAX_D == 64.0


# the project's half-precision gates against the fp32 model at 436 x 1024, 12 iterations (max-abs / mean-abs px)
HALF_GATES = {torch.float16: (8e-2, 2e-2), torch.bfloat16: (5e-1, 1e-1)}


def test_half_precision_at_full_size():
    sd = LO.synth_state_dict("lcv_raft", 5)
    img = torch.from_numpy(synth.synth_images(1, 436, 1024, 6, "smooth")).to(DEV)
    check_half_against_fp32(lambda dtype: _model("lcv_raft", sd, dtype, iters=12), img, HALF_GATES, "lcv_raft at 436x1024, 12 iterations")


def _half_errors(name, sd, img):
    errs = {}
    with torch.no_grad():
        ref = _model(name, sd, iters=12)({"images": img})["flows"].float()
        for dtype in HALF_GATES:
            e = (_model(name, sd, dtype, iters=12)({"images": img.to(dtype)})["flows_fp32"].float() - ref).abs()
            errs[dtype] = (e.max().item(), e.mean().item())
            print(f"{name} at 436x1024, 12 iterations, {dtype}: max-abs {errs[dtype][0]:.4f} mean-abs {errs[dtype][1]:.5f} px "
                  f"(max |flow| {ref.abs().max().item():.1f})")
    return errs


def test_half_precision_of_the_small_model_at_full_size():
    """lcv_raft_small misses the gates above, and so does raft_small on the same weights (DESIGN.md section 5, LCV): its error is
    raft_small's loop's.  Gate: within 1.5 times raft_small's own error on the same update block and encoders."""
    sd = LO.synth_state_dict("lcv_raft_small", 5)
    img = torch.from_numpy(synth.synth_images(1, 436, 1024, 6, "smooth")).to(DEV)
    lcv = _half_errors("lcv_raft_small", sd, img.flip(2))
    raft = _half_errors("raft_small", {k: v for k, v in sd.items() if not k.startswith("corr_block.")}, img)
    for dtype in HALF_GATES:
        assert lcv[dtype][0] < 1.5 * raft[dtype][0] + 0.02 and lcv[dtype][1] < 1.5 * raft[dtype][1] + 0.002, dtype


def test_tiny_grid_runs_where_raft_refuses():
    """32x32 frames (a 4x4 grid): RAFT's pyramid would have an empty level; LCV's never pools and runs, in every storage type."""
    sd = LO.synth_state_dict("lcv_raft", 414)
    img = torch.from_numpy(synth.synth_images(1, 32, 32, 424, "smooth")).to(DEV)
    g = load_golden("e2e_lcv_raft_tiny")[1]["flows"]
    for dtype, tol in ((torch.float16, 0.05), (torch.bfloat16, 0.4)):
        with torch.no_grad():
            out = _model("lcv_raft", sd, dtype, iters=3)({"images": img.to(dtype)})["flows_fp32"].float().cpu().numpy()
        assert np.abs(out - g).max() < tol
