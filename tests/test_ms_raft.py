"""CPU: MS-RAFT+.

The oracle's MS-RAFT+ stages (tests/ms_raft_oracle.py) against the reference's own outputs (tests/golden/op_ms_raft_p.npz,
e2e_ms_raft_p_*.npz and state_shapes_ms_raft_p.json, written by tests/make_ms_raft_golden.py), the model's parameter surface and
host-side checks, and the C-ABI exports and argument checks of the new kernels and loop.
"""
import ctypes as C
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

import ptlflow_b200  # noqa: F401  (before the reference shim below can put its own lightning stand-in into sys.modules)
import ms_raft_oracle as MS
from helpers import GOLDEN, load_golden, lib as _lib, raft_cfg
from oracle import raft_oracle as O
from oracle import ref_shim


@pytest.mark.parametrize("name", MS.E2E)
def test_ms_raft_e2e_matches_reference(name):
    recipe, g = load_golden(name)
    flow_init = torch.from_numpy(g["flow_init"]) if recipe["warm"] else None
    out = MS.forward_recipe(recipe, flow_init)
    assert out["flows"].shape == g["flows"].shape and out["flow_small"].shape == g["flow_small"].shape
    assert np.isfinite(g["flows"]).all() and np.abs(g["flows"]).max() > 0.5  # the fixture is not degenerate
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 2e-4
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 2e-4


def test_ms_raft_operators():
    g = np.load(os.path.join(GOLDEN, "op_ms_raft_p.npz"))
    sd, x = MS.op_inputs()
    with O.fp32_strict(), torch.no_grad():
        net, mask, delta = MS.update_block(x["net"], x["inp"], x["corr"], x["flow"], sd)
        outs = dict(block=MS.residual_block(x["block_in"], sd, "fnet.layer2.0.", 2),
                    up_layer=MS.up_layer(x["up_coarse"], x["up_skip"], sd, "fnet.up_layer1"), net=net, mask=mask, delta=delta,
                    up_flow=MS.convex_up2(x["coords"] - O.coords_grid(2, 6, 9), x["mask"]), up_coords=MS.convex_up2(x["coords"], x["mask"]))
    for k, v in outs.items():
        assert v.shape == g[k].shape, k
        assert np.abs(v.numpy() - g[k]).max() < 1e-4 * max(1.0, float(np.abs(g[k]).max())), k


def test_state_dict_contract():
    import ptlflow_b200 as pb

    with open(os.path.join(GOLDEN, "state_shapes_ms_raft_p.json")) as f:
        ref = {k: tuple(v) for k, v in json.load(f).items()}
    assert MS.state_dict_shapes() == ref
    m = pb.get_model("ms_raft_p")
    sd = m.state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert {k: tuple(v.shape) for k, v in sd.items()} == ref
    assert len(ref) == 302 and sum(p.numel() for p in m.parameters()) == 16177316
    res = m.load_state_dict(MS.synth_state_dict(ref, 1), strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    blk = m.fnet.layer2[0]
    assert blk.norm3 is blk.downsample[1]
    assert "cnet.layer4.0.norm3.weight" in sd and "cnet.layer4.0.downsample.1.weight" in sd


def test_checkpoint_loads_offline(tmp_path):
    import ptlflow_b200 as pb

    src = pb.get_model("ms_raft_p")
    ckpt = tmp_path / "ms_raft_p.ckpt"
    torch.save({"state_dict": MS.synth_state_dict(MS.state_dict_shapes(), 3)}, ckpt)
    m = pb.get_model("ms_raft_p", ckpt_path=str(ckpt))
    assert torch.equal(m.state_dict()["update_block.mask.2.weight"], MS.synth_state_dict(MS.state_dict_shapes(), 3)["update_block.mask.2.weight"])
    assert set(src.state_dict()) == set(m.state_dict())


def test_registry_and_defaults():
    import ptlflow_b200 as pb

    assert "ms_raft_p" in pb.get_model_names() and "ms_raft_p" in pb.get_trainable_model_names()
    m = pb.get_model("ms_raft_p")
    assert tuple(m.iters) == (4, 6, 5, 10) and m.lookup_pyramid_levels == 2 and m.lookup_radius == 4 and m.alternate_corr
    assert m.output_stride == 16 and m.correlation_depth == 162
    assert m.update_block.mask[2].out_channels == 36 and m.update_block.encoder.convc1.in_channels == 162
    assert set(m.pretrained_checkpoints) == {"mixed"}
    for k in ("gamma", "max_flow", "iters", "lookup_pyramid_levels", "lookup_radius", "alternate_corr"):
        assert hasattr(m.hparams, k), k
    m3 = pb.get_model("ms_raft_p", args=Namespace(model=Namespace(lookup_pyramid_levels=3, lookup_radius=3)))
    assert m3.corr_levels == 3 and m3.corr_radius == 3 and m3.update_block.encoder.convc1.in_channels == 3 * 49


@pytest.mark.parametrize("iters", [(4, 6, 5), (4, 6, 5, 10, 2), (4, 0, 5, 10), (1, 1, 1, -1), 7])
def test_bad_iters_raise(iters):
    import ptlflow_b200 as pb

    with pytest.raises(ValueError, match="iters"):
        pb.get_model("ms_raft_p", args=Namespace(model=Namespace(iters=iters)))
    m = pb.get_model("ms_raft_p")
    m.iters = iters
    with pytest.raises(ValueError, match="iters"):
        m._check_grid(4, 6)


def test_grid_and_warm_start_checks_on_the_host():
    import ptlflow_b200 as pb

    m = pb.get_model("ms_raft_p")
    m._check_grid(2, 2)
    with pytest.raises(ValueError, match="lookup_pyramid_levels"):
        m._check_grid(1, 6)
    pb.get_model("ms_raft_p", args=Namespace(model=Namespace(lookup_pyramid_levels=1)))._check_grid(1, 1)
    # the warm start is checked before anything touches the device (these CPU tensors would otherwise fail later, differently)
    img = torch.zeros(1, 2, 3, 100, 150)
    with pytest.raises(ValueError, match="multiples of 16"):
        m({"images": img, "prev_preds": {"flow_small": torch.zeros(1, 2, 6, 9)}})
    with pytest.raises(RuntimeError, match="CUDA"):
        m({"images": torch.zeros(1, 2, 3, 64, 96), "prev_preds": {"flow_small": torch.zeros(1, 2, 4, 6)}})


def test_volume_size_limit_raises():
    import ptlflow_b200 as pb

    m = pb.get_model("ms_raft_p", args=Namespace(model=Namespace(alternate_corr=False)))
    with pytest.raises(ValueError, match="alternate_corr=True"):
        m._check_volume(torch.zeros(1, 2, 3, 436, 1024))
    m._check_volume(torch.zeros(1, 2, 3, 128, 192))
    pb.get_model("ms_raft_p")._check_volume(torch.zeros(1, 2, 3, 436, 1024))


def test_c_abi_exports():
    L = _lib()
    lib = L.load()
    for sym in ("pfb_group_norm_act", "pfb_group_norm_apply", "pfb_upsample2x_concat", "pfb_convex_upsample2x", "pfb_downflow",
                "pfb_corr_lookup_onthefly_ex", "pfb_corr_lookup_onthefly_tc_ex", "pfb_msraft_workspace_bytes", "pfb_msraft_refine",
                "pfb_msraft_update_iter"):
        assert hasattr(lib, sym) and sym in L.SIGNATURES, sym


CFG = dict(dtype=2, B=2, H=16, W=24, feat_dim=256, corr_levels=2, corr_radius=4, hidden_dim=128, context_dim=128, iters=4,
           alternate_corr=1, out_h=32, out_w=48, num_heads=1)  # bf16


def test_msraft_entry_points_check_their_arguments():
    L = _lib()
    lib = L.load()
    cfg = lambda variant, **kw: C.byref(raft_cfg(L, CFG, variant=variant, **kw))  # noqa: E731
    n5 = lib.pfb_msraft_workspace_bytes(cfg(L.VARIANT_MS_RAFT_P))
    assert n5 > 0
    assert lib.pfb_msraft_workspace_bytes(cfg(L.VARIANT_RAFT)) == 0  # VARIANT_MS_RAFT_P only
    assert lib.pfb_raft_workspace_bytes(cfg(L.VARIANT_MS_RAFT_P)) == 0  # the raft, skflow and sea_raft loops refuse it
    assert lib.pfb_skflow_workspace_bytes(cfg(L.VARIANT_MS_RAFT_P)) == 0
    assert lib.pfb_searaft_workspace_bytes(cfg(L.VARIANT_MS_RAFT_P)) == 0
    assert lib.pfb_raft_workspace_bytes(cfg(L.VARIANT_RAFT)) > n5  # a 576-channel mask against a 36-channel one
    buf, w = L.RaftBuffers(), L.RaftWeights()
    assert lib.pfb_msraft_refine(cfg(L.VARIANT_RAFT), C.byref(w), C.byref(buf), 0.0, None, None) == -1
    assert b"variant" in lib.pfb_last_error()
    assert lib.pfb_raft_refine(cfg(L.VARIANT_MS_RAFT_P), C.byref(w), C.byref(buf), None) == -1
    assert lib.pfb_msraft_update_iter(cfg(L.VARIANT_RAFT_SMALL), C.byref(w), C.byref(buf), None, None, 0.0, None) == -1


def test_new_kernels_check_their_arguments():
    L = _lib()
    lib = L.load()
    # group norm: group size must divide C, C % 8, null pointers
    assert lib.pfb_group_norm_act(16, 16, None, 16, None, None, None, 1, 4, 4, 64, 7, 1e-5, 1, L.F16, None) == -1
    assert lib.pfb_group_norm_act(16, 16, None, 16, None, None, None, 1, 4, 4, 60, 4, 1e-5, 1, L.F16, None) == -1
    assert lib.pfb_group_norm_apply(None, 16, None, 16, None, None, None, 1, 4, 4, 64, 8, 1e-5, 1, L.F16, None) == -1
    # resize into the concat buffer: channel counts multiples of 8, 16-byte alignment
    assert lib.pfb_upsample2x_concat(16, 12, 16, 8, 16, 1, 4, 4, L.F16, None) == -1
    assert lib.pfb_upsample2x_concat(18, 16, 16, 8, 16, 1, 4, 4, L.F16, None) == -1
    # convex 2x: bad mode, window outside the upsampled grid
    assert lib.pfb_convex_upsample2x(16, 16, 16, 2, 1, 4, 4, 8, 8, 0, 0, L.F16, None) == -1
    assert lib.pfb_convex_upsample2x(16, 16, 16, 0, 1, 4, 4, 8, 8, 1, 0, L.F16, None) == -1
    assert lib.pfb_downflow(16, 16, 1, 4, 4, 0, 1, None) == -1
    # explicit lookup scales must not be negative
    pyr = (C.c_void_p * 2)(16, 16)
    assert lib.pfb_corr_lookup_onthefly_ex(16, pyr, 16, 16, 1, 8, 8, 128, 2, 4, -1.0, L.F16, L.F16, 0, 168, None) == -1
    assert lib.pfb_corr_lookup_onthefly_tc_ex(16, pyr, 16, 16, 16, 1, 8, 8, 128, 2, 4, -1.0, L.F16, 168, None) == -1


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout absent")
def test_live_reference_agrees_with_ms_raft_fixtures():
    """Where the reference checkout exists, re-run the real reference for two fixtures: they are not stale."""
    import make_ms_raft_golden as MG

    for name in ("e2e_ms_raft_p_default", "e2e_ms_raft_p_iters1212"):
        recipe, g = load_golden(name)
        out = MG.reference_e2e(recipe)
        assert np.abs(out["flows"] - g["flows"]).max() < 1e-5, name
