"""CPU: CRAFT -- the fp32 oracle against the reference's fixtures (and the live reference where its checkout exists), the state-dict
contract, the registry and defaults, every constructor and grid refusal, the analytic window bias against the reference's
SlidingPosBiases2D, the batch-global clamp of the clamp fixture, the identities the kernels rely on, and the C-ABI argument checks of
the a23 entry points."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import ptlflow_b200  # noqa: E402,F401  (imported before the reference's shim stubs lightning, so the models keep their hparams)
import craft_oracle as CR  # noqa: E402
from oracle import ref_shim  # noqa: E402
from helpers import check_live_reference, check_oracle_fixture, lib as _lib, load_golden  # noqa: E402

needs_reference = pytest.mark.skipif(not ref_shim.available(), reason="the reference checkout is not available")


@pytest.mark.parametrize("name", CR.E2E)
def test_craft_e2e_oracle_matches_reference(name):
    check_oracle_fixture(CR, name, 1e-4, 1e-4)


def test_clamp_fixture_is_batch_global():
    """In the clamp case exactly one sample's largest inter-frame score exceeds the clip, so the other sample is clamped only because
    the decision is taken over the whole batch; every other case stays below it."""
    for name in CR.E2E:
        g = load_golden(name)[1]
        if "max_score" not in g:
            continue
        over = int((g["max_score"] > CR.CLIP).sum())
        assert over == (1 if name == "e2e_craft_clamp" else 0), (name, g["max_score"])


@needs_reference
def test_craft_fixtures_match_live_reference():
    import make_craft_golden as MK

    check_live_reference(MK, CR, ["e2e_craft_ragged", "e2e_craft_modes"], 1e-5)


def test_state_dict_contract_and_checkpoints():
    import ptlflow_b200 as pb

    m = pb.get_model("craft")
    sd = m.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == CR.state_dict_shapes()
    assert len(sd) == 202 and sum(p.numel() for p in m.parameters()) == 6307435
    assert set(m.pretrained_checkpoints) == {"things", "sintel", "kitti"}
    assert m.corr_fn.setrans.key.weight is m.corr_fn.setrans.query.weight
    for kw in ({"inter_num_modes": 2, "intra_num_modes": 1, "f2_num_modes": 2, "pos_bias_radius": 3, "corr_radius": 3}, {"craft": False}):
        m = pb.get_model("craft", args=__import__("argparse").Namespace(model=__import__("argparse").Namespace(**kw)))
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == CR.state_dict_shapes(kw)
        m.load_state_dict(CR.synth_state_dict(kw, 1), strict=True)


def test_registry_and_defaults():
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib as L
    from ptlflow_b200.models.craft.craft import craft

    assert "craft" in pb.get_model_names()
    m = craft()
    assert (m.iters, m.corr_levels, m.corr_radius, m.f2_num_modes, m.inter_num_modes, m.intra_num_modes, m.pos_bias_radius) == (32, 4, 4, 4, 4, 4, 7)
    assert m._variant == L.VARIANT_GMA and m.hparams.gamma == 0.8
    assert craft(corr_radius=-1).corr_radius == 4 and craft(num_heads=8).num_heads == 8


@pytest.mark.parametrize("kw, match", [(dict(f2trans="none"), "f2trans"), (dict(f1trans="shared"), "f1trans"), (dict(f1trans="private"), "f1trans"),
                                       (dict(use_setrans=False), "use_setrans"), (dict(inter_pos_code_type="lsinu"), "bias"),
                                       (dict(intra_pos_code_type="sinu"), "bias"), (dict(corr_levels=3), "4 levels"), (dict(iters=0), "iters"),
                                       (dict(inter_num_modes=3), "inter_num_modes"), (dict(intra_num_modes=8), "intra_num_modes"),
                                       (dict(f2_num_modes=0), "f2_num_modes"), (dict(pos_bias_radius=16), "pos_bias_radius")])
def test_constructor_refusals(kw, match):
    from ptlflow_b200.models.craft.craft import craft

    with pytest.raises(ValueError, match=match):
        craft(**kw)


def test_grid_limit_raises_before_any_launch():
    from ptlflow_b200.models.craft.craft import craft

    m = craft()
    m._check_grid(200, 200)
    for h8, w8 in ((201, 20), (20, 201)):
        with pytest.raises(ValueError, match="200"):
            m._check_grid(h8, w8)


@needs_reference
@pytest.mark.parametrize("R, h, w", [(0, 5, 6), (2, 3, 4), (7, 6, 9), (3, 11, 9)])
def test_window_bias_matches_sliding_pos_biases(R, h, w):
    """The analytic bias biases[ky - qy + R][kx - qx + R] (0 outside the window) equals the reference's scattered table, read before
    its padding is cut (with R = 0 the reference's [R:-R] slice is empty; its table still holds the diagonal), on grids smaller and
    larger than the window."""
    import make_craft_golden as MK

    st = MK.load_craft().setrans
    g = torch.Generator().manual_seed(R * 100 + h)
    mod = st.SlidingPosBiases2D(2, R, max_pos_size=(12, 12))
    mod.biases.data.copy_(torch.randn(2 * R + 1, 2 * R + 1, generator=g))
    padded = torch.zeros(h, w, h + 2 * R, w + 2 * R)
    with torch.no_grad():
        padded[(mod.all_h1s[:h, :w], mod.all_w1s[:h, :w], mod.all_h2s[:h, :w], mod.all_w2s[:h, :w])] = mod.biases
        ref = padded[:, :, R:R + h, R:R + w].reshape(h * w, h * w)
        if R > 0:
            assert torch.equal(mod((1, 1, h, w), torch.float32, "cpu").reshape(h * w, h * w), ref)
        assert torch.equal(CR.window_bias(mod.biases.detach(), h, w), ref)


def test_mode_mix_identities():
    """The kernels drop feat2score's bias (softmax over modes is shift-invariant) and add the -1e9 mask where the reference does:
    both are exact in fp32."""
    g = torch.Generator().manual_seed(0)
    s = torch.randn(2, 4, 6, 6, generator=g) * 30
    sd = {"corr_fn.setrans.attn_softaggr.feat2score.weight": torch.tensor([[0.7]]), "corr_fn.setrans.attn_softaggr.feat2score.bias": torch.tensor([5.0])}
    mixed = CR.mode_mix(s, sd, 4)
    pi = torch.softmax(0.7 * s, dim=1)
    torch.testing.assert_close(mixed, (pi * s).sum(1), atol=1e-5, rtol=1e-6)
    assert torch.equal(CR.mode_mix(s[:, :1], sd, 1), s[:, 0])
    logits = torch.randn(36, 36, generator=g) + CR.chebyshev_mask(6, 6, 2)
    p = torch.softmax(logits, -1)
    assert torch.equal(p == 0, CR.chebyshev_mask(6, 6, 2) < 0)


def test_a23_argument_checks():
    L = _lib()
    lib = L.load()
    p = C.c_void_p(16)
    assert lib.pfb_craft_clamp_flag(None, 4, 100.0, p, 0, None) == -1
    assert lib.pfb_craft_clamp_flag(p, 0, 100.0, p, 0, None) == -1
    # (logits, rows, H, W, bias, R, mask_radius, flag, clip, dtype, stream)
    ok = [p, 20, 4, 5, p, 2, -1, p, 100.0, 1, None]
    for i, bad in ((0, None), (1, 21), (2, 201), (4, None), (5, 16), (5, -1), (7, None), (9, 3)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_craft_window_softmax(*args) == -1, (i, bad)
    # (feat, feat_stride, M, F, w, coeff, skip, skip_stride, skip_offset, out, out_stride, out_offset, P, dtype, stream)
    ok = [p, 512, 4, 128, p, 1.0, p, 256, 0, p, 256, 128, 10, 1, None]
    for i, bad in ((2, 5), (3, 64), (1, 511), (10, 255), (12, 0), (4, None)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_craft_mode_aggregate(*args) == -1, (i, bad)
    assert lib.pfb_craft_volume_workspace_bytes(1, 4, 5) >= 400 * 4 and lib.pfb_craft_volume_workspace_bytes(0, 4, 5) == 0
    # (scores, M, a, bias, R, flag, clip, level0, ws, ws_bytes, B, H, W, dtype, stream)
    ok = [p, 4, 0.5, p, 7, p, 100.0, p, p, 1 << 20, 1, 4, 5, 1, None]
    for i, bad in ((1, 5), (4, 16), (9, 16), (10, 0), (0, None)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_craft_volume_norm(*args) == -1, (i, bad)

    # (q1, k2, M, a, bias, R, flag, clip, pyramid, ws, ws_bytes, B, H, W, levels, dtype, stream)
    pyr = (C.c_void_p * 4)(16, 16, 16, 16)
    assert lib.pfb_craft_volume_tiled_workspace_bytes(1, 16, 20) > 0 and lib.pfb_craft_volume_tiled_workspace_bytes(0, 16, 20) == 0
    ok = [p, p, 4, 0.5, p, 7, p, 100.0, pyr, p, 1 << 20, 1, 16, 20, 4, 1, None]
    for i, bad in ((0, None), (1, C.c_void_p(8)), (2, 3), (5, 16), (10, 16), (14, 5), (12, 7), (15, 0)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_craft_volume_tiled(*args) == -1, (i, bad)
