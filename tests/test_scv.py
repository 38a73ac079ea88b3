"""CPU: SCV -- the fp32 oracle against the reference's fixtures (and the live reference where its checkout exists), the state-dict
contracts of scv4 / scv8, the constructor and grid checks, the encoders' projected shortcuts, and the C-ABI argument checks of the a21
entry points and loop variants VARIANT_SCV8 / VARIANT_SCV4."""
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

import scv_oracle as S  # noqa: E402
from oracle import ref_shim  # noqa: E402
from helpers import lib as _lib, raft_cfg  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


@pytest.mark.parametrize("name", S.E2E)
def test_scv_e2e_oracle_matches_reference(name):
    case = S.E2E_CASES[S.E2E.index(name)]
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    rec = S.recipe_of(case)
    assert json.loads(g["recipe"].tobytes()) == json.loads(json.dumps(rec))
    fi = torch.from_numpy(g["flow_init"]) if rec["warm"] else None
    out = S.forward_recipe(rec, fi)
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 2e-4
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 2e-4
    if rec["warm"]:
        first = S.forward_recipe(rec)
        assert np.abs(first["flow_small"].numpy() - g["prev_flow_small"]).max() < 2e-4


def test_scv_operators():
    g = np.load(os.path.join(GOLDEN, "op_scv.npz"))
    sds, x = S.op_inputs()
    with S.O.fp32_strict(), torch.no_grad():
        out = S.op_outputs(sds, x)
    assert np.array_equal(out["knn_idx"].numpy(), g["knn_idx"])
    for k, v in out.items():
        np.testing.assert_allclose(v.numpy(), g[k], atol=1e-5, rtol=0, err_msg=k)
    # the displacements the reference keeps are (ty - qy, tx - qx) of the selected targets
    p = S.OP_KNN
    np.testing.assert_array_equal(S.displacements(out["knn_idx"], p["H"], p["W"]).numpy(), g["knn_disp"])
    lk = g["lookup"]
    assert np.isfinite(lk).all()
    # displacement rows 0 / 1 of match 2 sit exactly on +-4 at level 0: the far corner carries weight 0, the bin on the edge the value
    assert lk[0, 0, 8 * 9 + 8] == pytest.approx(float(x["val"][0, 0, 2]), abs=1e-6)


@pytest.mark.skipif(not ref_shim.available(), reason="the reference checkout is not available")
def test_scv_fixtures_match_live_reference():
    import make_scv_golden as MK

    g = np.load(os.path.join(GOLDEN, "op_scv.npz"))
    for k, v in MK.reference_ops().items():
        np.testing.assert_allclose(v, g[k], atol=1e-6, rtol=0, err_msg=k)
    for name in ("e2e_scv4_ragged", "e2e_scv8_k8"):
        rec = S.recipe_of(S.E2E_CASES[S.E2E.index(name)])
        g = np.load(os.path.join(GOLDEN, name + ".npz"))
        assert np.abs(MK.reference_e2e(rec)["flows"] - g["flows"]).max() < 1e-6


@pytest.mark.parametrize("model", S.MODELS)
def test_state_dict_contract(model):
    import ptlflow_b200 as pb

    m = pb.get_model(model)
    sd = m.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == S.state_dict_shapes(model)
    assert len(sd) == 235 and tuple(sd["update_block.encoder.convc1.weight"].shape) == (256, 405, 1, 1)
    assert tuple(sd["update_block.mask.2.weight"].shape) == ((144 if model == "scv4" else 576), 256, 1, 1)
    # every residual block carries its projection, and batch norm's shared norm3 / downsample.1 keys
    assert "cnet.layer1.0.downsample.0.weight" in sd and "cnet.layer1.0.norm3.running_var" in sd and "cnet.layer3.1.downsample.1.weight" in sd
    m.load_state_dict(S.synth_state_dict(model, 1), strict=True)
    expect = {"chairs", "kitti", "sintel", "things"} if model == "scv4" else {"chairs", "things"}
    assert set(m.pretrained_checkpoints) == expect


def test_registry_and_defaults():
    import ptlflow_b200 as pb
    from ptlflow_b200 import get_trainable_model_names

    for model, variant in (("scv4", 10), ("scv8", 9)):
        assert model in pb.get_model_names() and model in get_trainable_model_names()
        m = pb.get_model(model)
        assert (m.num_k, m.iters, m.gamma, m.max_flow, m._variant, m.corr_levels, m.corr_radius) == (32, 32, 0.8, 400, variant, 5, 4)
    from ptlflow_b200.models.scv.scv import scv4

    m = scv4(num_k=8, iters=5)
    assert m.num_k == 8
    with pytest.raises(ValueError, match="num_k"):
        m.num_k = 40  # checked on every change, not only at construction
    m.num_k = 16
    assert m._extra_engine_args() == {"num_k": 16}


def test_raft_encoders_keep_their_identity_shortcuts():
    from ptlflow_b200.models.raft.extractor import BasicEncoder
    from ptlflow_b200.models.scv.scv import SCVEncoder, SCVEncoderQuarter

    raft_enc = BasicEncoder(256, "batch")
    assert raft_enc.layer1[0].downsample is None and raft_enc.layer2[0].downsample is not None
    q = SCVEncoderQuarter(256, "instance").eval()
    assert q.layer3[0].conv1.stride == (1, 1) and q.layer1[1].downsample is not None
    with torch.no_grad():
        x = torch.randn(1, 3, 32, 48)
        assert q(x).shape == (1, 256, 8, 12) and SCVEncoder(256, "instance").eval()(x).shape == (1, 256, 4, 6)


@pytest.mark.parametrize("kw, match", [(dict(num_k=0), "num_k"), (dict(num_k=33), "num_k"), (dict(iters=0), "iters")])
def test_constructor_refuses_what_the_kernels_cannot_run(kw, match):
    from ptlflow_b200.models.scv.scv import scv4, scv8

    for cls in (scv4, scv8):
        with pytest.raises(ValueError, match=match):
            cls(**kw)


def test_grid_smaller_than_num_k_raises():
    import ptlflow_b200 as pb

    m8, m4 = pb.get_model("scv8"), pb.get_model("scv4")
    with pytest.raises(ValueError, match="num_k=32"):
        m8._check_grid(4, 7)  # 28 pixels
    m8._check_grid(4, 8)
    m4._check_grid(2, 4)  # the 1/4 grid is 4 x 8
    with pytest.raises(ValueError, match="num_k=32"):
        m4._check_grid(1, 4)
    m8.num_k = 8
    m8._check_grid(2, 4)


CFG = dict(dtype=1, B=1, H=12, W=16, feat_dim=32, corr_levels=5, corr_radius=4, hidden_dim=128, context_dim=128, iters=2,
           alternate_corr=0, out_h=96, out_w=128, pad_top=0, pad_left=0, impl=0, volume_layout=0, fork_flow=0, num_heads=1)


def test_loop_variants_9_10_workspace_and_refusals():
    L = _lib()
    lib = L.load()
    cfg = dict(CFG, variant=L.VARIANT_SCV8)
    ws = lambda **kw: lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, cfg, **kw)))  # noqa: E731
    assert ws() > 0 and ws(variant=L.VARIANT_SCV4) > 0 and ws(feat_dim=1) == ws()
    for bad in (dict(corr_levels=4), dict(corr_radius=3), dict(alternate_corr=1), dict(volume_layout=1), dict(feat_dim=0),
                dict(feat_dim=33), dict(H=4, W=7), dict(hidden_dim=96)):
        assert ws(**bad) == 0, bad
        assert ws(variant=L.VARIANT_SCV4, **bad) == 0, bad
    assert ws(H=4, W=8) > 0 and ws(H=1, W=1, feat_dim=1) > 0  # no pyramid levels to fit: any grid with num_k pixels
    for sym in ("pfb_msraft_workspace_bytes", "pfb_ccmr_workspace_bytes", "pfb_skflow_workspace_bytes", "pfb_searaft_workspace_bytes"):
        assert getattr(lib, sym)(C.byref(raft_cfg(L, cfg))) == 0, sym
    # the lookup buffer: 405 planes, 408 in f16 (rows of 16 bytes), 405 in fp32; scv4's mask has 144 channels, scv8's 576
    P = 12 * 16
    r = lambda n: (n + 255) // 256 * 256  # noqa: E731
    assert ws() - ws(variant=L.VARIANT_RAFT, feat_dim=0, corr_levels=4) == r(P * 408 * 2) - r(P * 328 * 2)
    assert ws(dtype=0) - ws(variant=L.VARIANT_RAFT, feat_dim=0, corr_levels=4, dtype=0) == r(P * 405 * 4) - r(P * 324 * 4)
    assert ws() - ws(variant=L.VARIANT_SCV4) == r(P * 576 * 2) - r(P * 144 * 2)


def test_scv_argument_checks():
    L = _lib()
    lib = L.load()
    p = C.c_void_p(16)
    # (f1, f2, val, idx, workspace, workspace_bytes, B, N, C, k, scale, dtype, impl, stream)
    ok = [p, p, p, p, p, 1 << 20, 1, 99, 256, 32, C.c_float(0.0625), 1, 0, None]
    for i, bad in ((0, None), (3, None), (6, 0), (7, 31), (8, 0), (9, 0), (9, 33), (11, 5), (12, 3)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_knn_topk(*args) == -1, (i, bad)
    # impl 2 (wgmma) refuses fp32, a C it has no instance for, and unaligned features; the workspace query refuses what the call does
    for i, bad in ((11, 0), (8, 96), (8, 320), (0, C.c_void_p(18))):
        args = list(ok)
        args[i], args[12] = bad, 2
        assert lib.pfb_knn_topk(*args) == -1, (i, bad)
        wargs = [args[0], args[1], args[6], args[7], args[8], args[9], args[11], 2]
        assert lib.pfb_knn_topk_workspace_bytes(*wargs) == 0, (i, bad)
    # (val, idx, coords, table, B, H, W, k, stream)
    ok = [p, p, p, p, 1, 4, 8, 32, None]
    for i, bad in ((0, None), (3, None), (5, 0), (6, 7), (7, 0), (7, 33)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_sparse_prepare(*args) == -1, (i, bad)
    # (table, coords, out, B, H, W, k, dtype, out_stride, stream)
    ok = [p, p, p, 1, 4, 8, 32, 1, 408, None]
    for i, bad in ((0, None), (2, None), (4, 0), (6, 0), (6, 33), (7, 9), (8, 404)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_sparse_lookup(*args) == -1, (i, bad)
    # (coords, mask, out, flow_small, B, H, W, out_h, out_w, pad_top, pad_left, dtype, stream): the window lies in 4H x 4W
    assert lib.pfb_convex_upsample4x(p, p, p, p, 1, 8, 8, 33, 32, 0, 0, 1, None) == -1
    assert lib.pfb_convex_upsample4x(p, p, p, p, 1, 8, 8, 32, 32, 1, 0, 1, None) == -1
