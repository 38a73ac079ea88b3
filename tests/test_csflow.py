"""CPU: CSFlow -- the fp32 oracle against the reference's fixtures (and the live reference where its checkout exists), the state-dict
contract, the constructor and grid checks, the convc1 permutation, and the C-ABI argument checks of the a20 entry points and loop
variant VARIANT_CSFLOW."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import csflow_oracle as CS  # noqa: E402
from oracle import ref_shim  # noqa: E402
from helpers import lib as _lib, raft_cfg  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


@pytest.mark.parametrize("name", CS.E2E)
def test_csflow_e2e_oracle_matches_reference(name):
    case = CS.E2E_CASES[CS.E2E.index(name)]
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    rec = CS.recipe_of(case)
    assert json.loads(g["recipe"].tobytes()) == json.loads(json.dumps(rec))
    fi = torch.from_numpy(g["flow_init"]) if rec["warm"] else None
    out = CS.forward_recipe(rec, fi)
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 1e-5
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 1e-5
    if rec["warm"]:
        first = CS.forward_recipe(rec)
        assert np.abs(first["flow_small"].numpy() - g["prev_flow_small"]).max() < 1e-5


def test_csflow_operators():
    g = np.load(os.path.join(GOLDEN, "op_csflow.npz"))
    sd, x = CS.op_inputs()
    with CS.O.fp32_strict(), torch.no_grad():
        out = CS.op_outputs(sd, x)
    for k, v in out.items():
        np.testing.assert_allclose(v.numpy(), g[k], atol=1e-5, rtol=0, err_msg=k)
    lk = g[f"lookup_r{CS.OP_LOOKUP_RADIUS}"]
    # the far-out-of-range coordinates read nothing, and nothing is NaN
    assert np.isfinite(lk).all() and not lk[0, :, 0, :2].any()
    # the softmax weights of the initial flow are exactly 1: corr_init is the plain sums
    init = torch.stack([out["sh"].sum(-1), out["sw"].sum(-1)], 1)
    assert torch.allclose(init, out["corr_init"], atol=1e-6, rtol=0)


@pytest.mark.skipif(not ref_shim.available(), reason="the reference checkout is not available")
def test_csflow_fixtures_match_live_reference():
    import make_csflow_golden as MK

    g = np.load(os.path.join(GOLDEN, "op_csflow.npz"))
    for k, v in MK.reference_ops().items():
        np.testing.assert_allclose(v, g[k], atol=1e-6, rtol=0, err_msg=k)
    rec = CS.recipe_of(CS.E2E_CASES[CS.E2E.index("e2e_csflow_r6")])
    g = np.load(os.path.join(GOLDEN, "e2e_csflow_r6.npz"))
    assert np.abs(MK.reference_e2e(rec)["flows"] - g["flows"]).max() < 1e-5


def test_state_dict_contract():
    import ptlflow_b200 as pb

    m = pb.get_model("csflow")
    sd = m.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == CS.state_dict_shapes()
    assert len(sd) == 203 and tuple(sd["update_block.encoder.convc1.weight"].shape) == (256, 648, 1, 1)
    for blk in ("conv1_1", "conv1_2", "conv2_1", "conv2_2"):
        assert f"strip_corr_block_v2.{blk}.conv.weight" in sd and f"strip_corr_block_v2.{blk}.bn.running_var" in sd
    m.load_state_dict(CS.synth_state_dict(4, 1), strict=True)
    assert set(m.pretrained_checkpoints) == {"chairs", "things", "kitti"}


def test_registry_and_defaults():
    import ptlflow_b200 as pb
    from ptlflow_b200 import get_trainable_model_names

    assert "csflow" in pb.get_model_names() and "csflow" in get_trainable_model_names()
    m = pb.get_model("csflow")
    assert (m.iters, m.corr_levels, m.corr_radius, m.dropout, m.gen_fmap, m.skip_encode) == (32, 4, 4, 0.0, False, False)
    assert (m.gamma, m.max_flow, m._variant) == (0.8, 400, 8)
    from ptlflow_b200.models.csflow.csflow import csflow

    m = csflow(corr_radius=3, iters=5)
    assert m.update_block.encoder.convc1.in_channels == 2 * 4 * 49 and m.iters == 5


@pytest.mark.parametrize("kw, match", [
    (dict(corr_levels=3), "4 levels"),
    (dict(corr_levels=5), "4 levels"),
    (dict(gen_fmap=True), "gen_fmap"),
    (dict(skip_encode=True), "skip_encode"),
    (dict(iters=0), "iters"),
    (dict(corr_radius=16), "corr_radius"),
])
def test_constructor_refuses_what_the_kernels_cannot_run(kw, match):
    from ptlflow_b200.models.csflow.csflow import csflow

    with pytest.raises(ValueError, match=match):
        csflow(**kw)


@pytest.mark.parametrize("h, w", [(96, 128), (128, 96), (120, 1024), (16, 16)])
def test_grid_limits_raise_before_any_launch(h, w):
    """1/8 grids (after padding) under 16 pixels per side, where the reference's coarsest level has one pixel and it returns NaN."""
    import ptlflow_b200 as pb

    m = pb.get_model("csflow").eval()
    with pytest.raises(ValueError, match="csflow needs"):
        m._check_grid(-(-h // 8), -(-w // 8))
    m._check_grid(16, 16)
    m._check_grid(-(-121 // 8), 128)


@pytest.mark.parametrize("radius", [0, 1, 4])
def test_convc1_permutation_round_trips(radius):
    """The packed convc1 over [4D taps of every level | strip taps of every level] equals the reference's convc1 over its per-level
    interleave [4D l | strip l], exactly (a 1x1 convolution is a sum over input columns)."""
    from ptlflow_b200.engine import csflow_convc1_permutation

    kk = (2 * radius + 1) ** 2
    perm = csflow_convc1_permutation(4, radius)
    assert sorted(perm.tolist()) == list(range(8 * kk))
    g = torch.Generator().manual_seed(radius)
    ref_corr = torch.randn(2, 8 * kk, 3, 4, generator=g, dtype=torch.float64)  # reference order
    w = torch.randn(5, 8 * kk, 1, 1, generator=g, dtype=torch.float64)
    # the buffer's order: all 4D levels, then all strip levels
    lv = ref_corr.view(2, 4, 2, kk, 3, 4)
    buf = torch.cat([lv[:, :, 0].reshape(2, 4 * kk, 3, 4), lv[:, :, 1].reshape(2, 4 * kk, 3, 4)], 1)
    assert torch.equal(buf, ref_corr[:, perm])
    torch.testing.assert_close(torch.nn.functional.conv2d(buf, w[:, perm]), torch.nn.functional.conv2d(ref_corr, w), rtol=1e-12, atol=1e-12)


CFG = dict(dtype=1, B=1, H=16, W=20, feat_dim=0, corr_levels=4, corr_radius=4, hidden_dim=128, context_dim=128, iters=2,
           alternate_corr=0, out_h=128, out_w=160, pad_top=0, pad_left=0, impl=0, volume_layout=1, fork_flow=0, num_heads=1)


def test_loop_variant8_workspace_and_refusals():
    L = _lib()
    lib = L.load()
    cfg = dict(CFG, variant=L.VARIANT_CSFLOW)
    ws = lambda **kw: lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, cfg, **kw)))  # noqa: E731
    assert ws() > 0 and ws(volume_layout=0) == ws() and ws(corr_radius=15) > ws() and ws(corr_radius=0) > 0
    for bad in (dict(corr_levels=3), dict(corr_levels=5), dict(alternate_corr=1), dict(volume_layout=2), dict(corr_radius=16),
                dict(hidden_dim=96), dict(volume_layout=1, dtype=0)):
        assert ws(**bad) == 0, bad
    # VARIANT_CSFLOW is a pfb_raft loop only
    for sym in ("pfb_msraft_workspace_bytes", "pfb_ccmr_workspace_bytes", "pfb_skflow_workspace_bytes", "pfb_searaft_workspace_bytes"):
        assert getattr(lib, sym)(C.byref(raft_cfg(L, cfg))) == 0, sym
    # the lookup buffer: 2 x 4 x 81 = 648 planes (already a multiple of 8); the rest of the workspace is VARIANT_RAFT's (324 planes)
    ref0 = ws(variant=L.VARIANT_RAFT)
    P = 16 * 20
    assert ws() - ref0 == (P * 648 * 2 + 255) // 256 * 256 - (P * 328 * 2 + 255) // 256 * 256
    assert ws(dtype=0, volume_layout=0) - ws(variant=L.VARIANT_RAFT, dtype=0, volume_layout=0) == (P * 648 * 4 + 255) // 256 * 256 - (P * 324 * 4 + 255) // 256 * 256


def test_strip_argument_checks():
    L = _lib()
    lib = L.load()
    p = C.c_void_p(16)
    assert lib.pfb_strip_table_width(20, 4) == 20 + 10 + 5 + 2 and lib.pfb_strip_table_width(17, 4) == 17 + 8 + 4 + 2
    assert lib.pfb_strip_table_width(7, 4) == 0 and lib.pfb_strip_table_width(8, 0) == 0
    # (gw, gh, kw, kh, B, H, W, C, dtype, stream)
    ok = [p, p, p, p, 1, 16, 20, 256, 1, None]
    for i, bad in ((0, None), (3, None), (4, 0), (7, 0), (8, 5)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_strip_means(*args) == -1, (i, bad)
    # (sw, sh, tab_w, tab_h, coords, B, H, W, levels, dtype, stream)
    ok = [p, p, p, p, p, 1, 16, 20, 4, 1, None]
    for i, bad in ((0, None), (3, None), (6, 7), (7, 7), (8, 0), (8, 9), (9, 3)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_strip_prepare(*args) == -1, (i, bad)
    # (tab_w, tab_h, coords, out, B, H, W, levels, radius, dtype, out_stride, out_offset, stream)
    ok = [p, p, p, p, 1, 16, 20, 4, 4, 1, 648, 324, None]
    for i, bad in ((2, None), (8, 16), (8, -1), (10, 647), (11, 325), (11, -1), (7, 5), (9, 4)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_strip_lookup(*args) == -1, (i, bad)
