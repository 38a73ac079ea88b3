"""CPU: Flow1D -- the fp32 oracle against the reference's fixtures (and the live reference where its checkout exists), the state-dict
contract, the constructor and grid checks, and the C-ABI argument checks of the a19 entry points and loop variant VARIANT_FLOW1D."""
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

import flow1d_oracle as FD  # noqa: E402
from oracle import ref_shim  # noqa: E402
from helpers import lib as _lib, raft_cfg  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


@pytest.mark.parametrize("name", FD.E2E)
def test_flow1d_e2e_oracle_matches_reference(name):
    case = FD.E2E_CASES[FD.E2E.index(name)]
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    rec = FD.recipe_of(case)
    assert json.loads(g["recipe"].tobytes()) == json.loads(json.dumps(rec))
    fi = torch.from_numpy(g["flow_init"]) if rec["warm"] else None
    out = FD.forward_recipe(rec, fi)
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 2e-4
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 2e-4
    if rec["warm"]:
        first = FD.forward_recipe(rec)
        assert np.abs(first["flow_small"].numpy() - g["prev_flow_small"]).max() < 2e-4


def _oracle_ops():
    sd, x = FD.op_inputs()
    f1, f2 = x["f1"], x["f2"]
    with torch.no_grad():
        pos = FD.position(6, 9, 256)
        cx, cy, f2_x, f2_y = FD.correlation(sd, f1, f2)
        out = {"position": pos, "attn_x": f2_x, "attn_y": f2_y}
        for r in (1, FD.OP_RADIUS, 32):
            lk = FD.lookup(cx, cy, x["coords"], r)
            out[f"lookup_x_r{r}"], out[f"lookup_y_r{r}"] = lk[:, : 2 * r + 1], lk[:, 2 * r + 1:]
        net, mask, delta = FD.O.basic_update_block(x["net"], x["inp"], x["corr"], x["flow"], sd)
        out.update(net=net, mask=mask, delta=delta)
    return out


def test_flow1d_operators():
    g = np.load(os.path.join(GOLDEN, "op_flow1d.npz"))
    with FD.O.fp32_strict():
        out = _oracle_ops()
    for k, v in out.items():
        np.testing.assert_allclose(v.numpy(), g[k], atol=1e-5, rtol=0, err_msg=k)
    # the far-out-of-range coordinates read nothing, and nothing is NaN
    assert np.isfinite(g["lookup_x_r32"]).all() and not g["lookup_x_r32"][0, :, 0, :2].any()


@pytest.mark.skipif(not ref_shim.available(), reason="the reference checkout is not available")
def test_flow1d_fixtures_match_live_reference():
    import make_flow1d_golden as MK

    g = np.load(os.path.join(GOLDEN, "op_flow1d.npz"))
    for k, v in MK.reference_ops().items():
        np.testing.assert_allclose(v, g[k], atol=1e-6, rtol=0, err_msg=k)
    rec = FD.recipe_of(FD.E2E_CASES[FD.E2E.index("e2e_flow1d_r8")])
    g = np.load(os.path.join(GOLDEN, "e2e_flow1d_r8.npz"))
    assert np.abs(MK.reference_e2e(rec)["flows"] - g["flows"]).max() < 1e-5


def test_state_dict_contract():
    import ptlflow_b200 as pb

    m = pb.get_model("flow1d")
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == FD.state_dict_shapes()
    assert sum(p.numel() for p in m.parameters()) == 5734208
    m.load_state_dict(FD.synth_state_dict(32, 1), strict=True)
    assert set(m.pretrained_checkpoints) == {"chairs", "things", "sintel", "kitti", "highres"}


def test_registry_and_defaults():
    import ptlflow_b200 as pb
    from ptlflow_b200 import get_trainable_model_names

    assert "flow1d" in pb.get_model_names() and "flow1d" in get_trainable_model_names()
    m = pb.get_model("flow1d")
    assert (m.iters, m.corr_radius, m.feature_channels, m.downsample_factor) == (32, 32, 256, 8)
    from ptlflow_b200.models.flow1d.flow1d import flow1d

    m = flow1d(corr_radius=8, feature_channels=128, iters=5)
    assert m.update_block.encoder.convc1.in_channels == 34 and m.attn_x.query_conv.in_channels == 128 and m.iters == 5


@pytest.mark.parametrize("kw, match", [
    (dict(downsample_factor=4), "downsample_factor"),
    (dict(hidden_dim=96), "hidden_dim"),
    (dict(context_dim=64), "context_dim"),
    (dict(feature_channels=96), "feature_channels"),
    (dict(feature_channels=320), "feature_channels"),
    (dict(corr_radius=65), "corr_radius"),
    (dict(corr_radius=0), "corr_radius"),
    (dict(iters=0), "iters"),
])
def test_constructor_refuses_what_the_kernels_cannot_run(kw, match):
    from ptlflow_b200.models.flow1d.flow1d import flow1d

    with pytest.raises(ValueError, match=match):
        flow1d(**kw)


@pytest.mark.parametrize("h, w", [(8, 64), (64, 8), (16, 8200), (8200, 16)])
def test_grid_limits_raise_before_any_launch(h, w):
    """1/8 grids (after padding) below 2 or above ATTN1D_MAX_L pixels per side: forward() checks the grid before anything runs."""
    import ptlflow_b200 as pb

    m = pb.get_model("flow1d").eval()
    with pytest.raises(ValueError, match="flow1d needs"):
        m._check_grid(-(-h // 8), -(-w // 8))
    m._check_grid(2, _lib().ATTN1D_MAX_L)


CFG = dict(dtype=1, B=1, H=8, W=12, feat_dim=0, corr_levels=1, corr_radius=32, hidden_dim=128, context_dim=128, iters=2,
           alternate_corr=0, out_h=64, out_w=96, pad_top=0, pad_left=0, impl=0, volume_layout=0, fork_flow=0, num_heads=1)


def test_loop_variant7_workspace_and_refusals():
    L = _lib()
    lib = L.load()
    cfg = dict(CFG, variant=L.VARIANT_FLOW1D)
    ws = lambda **kw: lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, cfg, **kw)))  # noqa: E731
    assert ws() > 0 and ws(corr_radius=64) > ws() and ws(corr_radius=1) > 0
    for bad in (dict(corr_radius=65), dict(corr_levels=2), dict(alternate_corr=1), dict(volume_layout=1), dict(H=1), dict(W=1),
                dict(hidden_dim=96)):
        assert ws(**bad) == 0, bad
    # the radius limit of the other loops is unchanged; VARIANT_FLOW1D is not a pfb_msraft / pfb_ccmr loop
    assert ws(variant=L.VARIANT_RAFT, corr_levels=4, corr_radius=16) == 0 and ws(variant=L.VARIANT_RAFT, corr_levels=4, corr_radius=4) > 0
    assert lib.pfb_msraft_workspace_bytes(C.byref(raft_cfg(L, cfg))) == 0 and lib.pfb_ccmr_workspace_bytes(C.byref(raft_cfg(L, cfg))) == 0
    # the lookup buffer: 2 (2r+1) = 130 planes, stride 136 in f16 (the rest of the workspace is VARIANT_RAFT's)
    ref0 = ws(variant=L.VARIANT_RAFT, corr_levels=1, corr_radius=4)  # 81 planes, stride 88
    P = 8 * 12
    assert ws() - ref0 == (P * 136 * 2 + 255) // 256 * 256 - (P * 88 * 2 + 255) // 256 * 256


def test_attn1d_and_lookup_argument_checks():
    L = _lib()
    lib = L.load()
    p = C.c_void_p(16)
    # (q, qs, k, ks, v, vs, out, os, B, H, W, C, axis, mode, scale, dtype, impl, stream)
    ok = [p, 256, p, 256, p, 256, p, 256, 1, 8, 12, 256, 0, L.ATTN1D_ATTN, 0.0625, 1, 0, None]
    for i, bad in ((11, 96), (11, 320), (12, 2), (13, 3), (15, 7), (10, L.ATTN1D_MAX_L + 1), (1, 128), (7, 128), (4, None), (8, 0),
                   (16, 3), (16, -1)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_attn1d(*args) == -1, (i, bad)
    args = list(ok)
    args[4], args[13] = None, L.ATTN1D_CORR  # the correlation needs no v
    args[9] = L.ATTN1D_MAX_L + 1  # ... and a column sequence may not exceed the limit either
    args[12] = 1
    assert lib.pfb_attn1d(*args) == -1
    # impl 2 (wgmma) refuses what it cannot run: fp32, C = 192, a pixel stride that is not a multiple of 8 elements
    for i, bad in ((15, 0), (11, 192), (1, 260)):
        args = list(ok)
        args[16], args[i] = 2, bad
        if i == 11:
            args[1] = args[3] = args[5] = args[7] = 192
        assert lib.pfb_attn1d(*args) == -1, (i, bad)
    # (corr_x, corr_y, coords, out, B, H, W, radius, dtype, out_stride, stream)
    ok = [p, p, p, p, 1, 8, 12, 32, 1, 136, None]
    for i, bad in ((7, 0), (7, 65), (9, 129), (8, 5), (0, None), (5, 0)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_corr1d_lookup(*args) == -1, (i, bad)
