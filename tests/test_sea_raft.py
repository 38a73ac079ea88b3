"""CPU: SEA-RAFT.

The oracle's SEA-RAFT stages (tests/sea_raft_oracle.py) against the reference's own outputs (tests/golden/op_sea_raft.npz,
e2e_sea_raft_*.npz and state_shapes_sea_raft*.json, written by tests/make_sea_raft_golden.py), the identity between the
reference's correlation pyramid and RAFT's pooled one, the model's parameter surface and hyperparameter checks, and the C-ABI
exports of the new kernel and loop.
"""
import ctypes as C
import json
import os
import re
from argparse import Namespace

import numpy as np
import pytest
import torch

import ptlflow_b200  # noqa: F401  (before the reference shim below can put its own lightning stand-in into sys.modules)
import sea_raft_oracle as SR
from helpers import GOLDEN, load_golden, lib as _lib, raft_cfg
from oracle import raft_oracle as O
from oracle import ref_shim, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", SR.E2E)
def test_sea_raft_e2e_matches_reference(name):
    recipe, g = load_golden(name)
    out = SR.forward_recipe(recipe)
    assert out["flows"].shape == g["flows"].shape
    assert np.isfinite(g["flows"]).all() and np.abs(g["flows"]).max() > 0.5  # the fixture is not degenerate
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 2e-4
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 2e-4


@pytest.mark.parametrize("b,h,w", SR.OP_GRIDS)
def test_sea_raft_operators(b, h, w):
    g = np.load(os.path.join(GOLDEN, "op_sea_raft.npz"))
    sd, net, inp, corr, flow = SR.op_inputs(b, h, w)
    x = torch.cat([net, inp, corr[:, :126], flow], 1)
    outs = [SR.convnext_block(x, sd, "update_block.refine.0.")] + list(SR.iteration(net, inp, corr, flow, sd))
    for key, arr in zip(("block", "net", "delta", "mask"), outs):
        flat = arr.numpy().reshape(-1)
        assert np.abs(flat[SR.op_sample(flat.size)] - g[f"{key}_{h}x{w}"]).max() < 1e-4, key


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout absent")
@pytest.mark.parametrize("levels,radius,h,w", [(4, 4, 16, 24), (4, 4, 17, 21), (3, 3, 13, 17), (1, 2, 3, 5)])
def test_reference_corr_block_is_the_pooled_pyramid(levels, radius, h, w):
    """SEA-RAFT's CorrBlock (one GEMM per level against a bilinearly halved fmap2) == RAFT's volume pooled 2x2 level by level, and
    its lookup is RAFT's: the identity the SEA-RAFT loop rests on."""
    import make_sea_raft_golden as MS

    MS.load_sea_raft()
    import ptlflow.models.sea_raft.corr as rc

    f1 = torch.from_numpy(synth.synth_normal("srcorr/f1", (2, 64, h, w), 7))
    f2 = torch.from_numpy(synth.synth_normal("srcorr/f2", (2, 64, h, w), 8))
    coords = O.coords_grid(2, h, w) + torch.from_numpy(synth.synth_normal("srcorr/d", (2, 2, h, w), 9, scale=3.0))
    ref = rc.CorrBlock(f1, f2, num_levels=levels, radius=radius)(coords)
    mine = O.corr_lookup(O.corr_pyramid(O.corr_volume(f1, f2), levels), coords, radius)
    assert ref.shape == mine.shape
    assert (ref - mine).abs().max().item() < 1e-5


def test_state_dict_contract():
    import ptlflow_b200 as pb

    for fname, name, kw in (("state_shapes_sea_raft.json", "sea_raft", {}), ("state_shapes_sea_raft_m.json", "sea_raft_m", {}),
                            ("state_shapes_sea_raft_iters0.json", "sea_raft", {"iters": 0})):
        with open(os.path.join(GOLDEN, fname)) as f:
            ref = {k: tuple(v) for k, v in json.load(f).items()}
        assert SR.state_dict_shapes(SR.PRETRAIN[name], kw.get("iters", 4)) == ref, fname
        m = pb.get_model(name, args=Namespace(model=Namespace(**kw)))
        sd = m.state_dict()
        assert list(sd.keys()) == list(ref.keys()), fname
        assert {k: tuple(v.shape) for k, v in sd.items()} == ref, fname
        res = m.load_state_dict(SR.synth_state_dict(ref, 1), strict=True)
        assert not res.missing_keys and not res.unexpected_keys
    assert len(ref) == 127
    m = pb.get_model("sea_raft")
    blk = m.cnet.layer2[0]
    assert blk.bn3 is blk.downsample[1]  # one module under two key paths, as the reference registers it
    assert "cnet.layer2.0.bn3.running_var" in m.state_dict() and "cnet.layer2.0.downsample.1.running_var" in m.state_dict()


def test_registry_and_defaults():
    import ptlflow_b200 as pb

    names = pb.get_trainable_model_names()
    expect = {"sea_raft": ("resnet18", 4, 276), "sea_raft_s": ("resnet18", 4, 276), "sea_raft_m": ("resnet34", 4, 472),
              "sea_raft_l": ("resnet34", 12, 472)}
    for name, (pretrain, iters, ntensors) in expect.items():
        assert name in names
        m = pb.get_model(name)
        assert (m.pretrain, m.iters, len(m.state_dict())) == (pretrain, iters, ntensors), name
        assert m.hparams.pretrain == pretrain and m.hparams.iters == iters
        if name != "sea_raft":
            assert set(m.pretrained_checkpoints) == {"tartan", "chairs", "things", "sintel", "kitti", "spring"}
    hp = pb.get_model("sea_raft").hparams
    for k in ("corr_levels", "corr_radius", "dim", "initial_dim", "num_blocks", "block_dims", "pretrain", "gamma", "max_flow", "iters",
              "alternate_corr", "use_var", "var_min", "var_max"):
        assert hasattr(hp, k), k


@pytest.mark.parametrize("dims", [(64, 128, 256), [64, 128, 256], [32, 64, 128]])
def test_block_dims_accepted_and_not_mutated(dims):
    import ptlflow_b200 as pb

    before = list(dims)
    m = pb.get_model("sea_raft", args=Namespace(model=Namespace(block_dims=dims)))
    assert list(dims) == before and type(m.hparams.block_dims) is type(dims)
    assert m.cnet.final_conv.in_channels == dims[2]


@pytest.mark.parametrize("kw,match", [(dict(dim=96), "dim"), (dict(pretrain="resnet50"), "pretrain")])
def test_bad_hyperparameters_raise(kw, match):
    import ptlflow_b200 as pb

    with pytest.raises(ValueError, match=match):
        pb.get_model("sea_raft", args=Namespace(model=Namespace(**kw)))


def test_grid_limit_is_checked_on_the_host():
    import ptlflow_b200 as pb

    m = pb.get_model("sea_raft")
    m._check_grid(16, 16)
    with pytest.raises(ValueError, match="2\\*\\*corr_levels"):
        m._check_grid(8, 12)
    pb.get_model("sea_raft", args=Namespace(model=Namespace(corr_levels=3)))._check_grid(8, 12)
    pb.get_model("sea_raft", args=Namespace(model=Namespace(iters=0)))._check_grid(8, 12)


def test_c_abi_exports_and_mirrors():
    L = _lib()
    lib = L.load()
    for sym in ("pfb_depthwise_conv_layernorm", "pfb_searaft_workspace_bytes", "pfb_searaft_refine", "pfb_searaft_update_iter"):
        assert hasattr(lib, sym) and sym in L.SIGNATURES
    text = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "ptlflow_b200.h")).read(), flags=re.S)
    for struct, mirror in (("pfb_convnext_block", L.ConvNextBlock), ("pfb_searaft_weights", L.SearaftWeights)):
        body = re.search(r"typedef\s+struct\s*\{([^{}]*)\}\s*" + struct + r"\s*;", text, flags=re.S).group(1)
        fields = [f for decl in body.split(";") if decl.strip() for f in re.findall(r"(\w+)\s*(?:\[[^\]]*\])?\s*(?:,|$)", decl.strip())]
        assert fields == [f[0] for f in mirror._fields_], struct
    assert int(re.search(r"#define\s+PFB_SR_MAX_BLOCKS\s+(\d+)", text).group(1)) == L.PFB_SR_MAX_BLOCKS


CFG = dict(dtype=2, B=2, H=16, W=24, feat_dim=256, corr_levels=4, corr_radius=4, hidden_dim=128, context_dim=128, iters=4, out_h=128,
           out_w=192, num_heads=1)  # bf16


def test_searaft_entry_points_check_their_arguments():
    L = _lib()
    lib = L.load()
    cfg = lambda variant, **kw: C.byref(raft_cfg(L, CFG, variant=variant, **kw))  # noqa: E731
    assert lib.pfb_searaft_workspace_bytes(cfg(L.VARIANT_SEA_RAFT)) > 0
    assert 0 < lib.pfb_searaft_workspace_bytes(cfg(L.VARIANT_SEA_RAFT, iters=0)) < lib.pfb_searaft_workspace_bytes(cfg(L.VARIANT_SEA_RAFT))
    assert lib.pfb_searaft_workspace_bytes(cfg(L.VARIANT_SKFLOW)) == 0  # VARIANT_SEA_RAFT only
    assert lib.pfb_raft_workspace_bytes(cfg(L.VARIANT_SEA_RAFT)) == 0  # the raft and skflow loops keep refusing it
    assert lib.pfb_skflow_workspace_bytes(cfg(L.VARIANT_SEA_RAFT)) == 0
    buf, w = L.RaftBuffers(), L.SearaftWeights()
    assert lib.pfb_searaft_refine(cfg(L.VARIANT_SKFLOW), C.byref(w), C.byref(buf), None) == -1
    assert b"variant" in lib.pfb_last_error()
    assert lib.pfb_raft_refine(cfg(L.VARIANT_SEA_RAFT), C.byref(L.RaftWeights()), C.byref(buf), None) == -1
    assert lib.pfb_skflow_refine(cfg(L.VARIANT_SEA_RAFT), C.byref(L.SkflowWeights()), C.byref(buf), None) == -1


def test_depthwise_layernorm_argument_checks():
    L = _lib()
    lib = L.load()
    # even kernel, k > 31, odd channel count, C > 512, odd offset, eps <= 0
    assert lib.pfb_depthwise_conv_layernorm(16, 384, 0, 16, 384, 0, 16, 16, 1, 8, 8, 384, 4, 1e-6, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_layernorm(16, 384, 0, 16, 384, 0, 16, 16, 1, 8, 8, 384, 33, 1e-6, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_layernorm(16, 384, 0, 16, 384, 0, 16, 16, 1, 8, 8, 383, 7, 1e-6, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_layernorm(16, 1024, 0, 16, 1024, 0, 16, 16, 1, 8, 8, 514, 7, 1e-6, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_layernorm(16, 384, 1, 16, 384, 0, 16, 16, 1, 8, 8, 382, 7, 1e-6, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_layernorm(16, 384, 0, 16, 384, 0, 16, 16, 1, 8, 8, 384, 7, 0.0, L.BF16, None) == -1


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout absent")
def test_live_reference_agrees_with_sea_raft_fixtures():
    """Where the reference checkout exists, re-run the real reference for two fixtures: they are not stale."""
    import make_sea_raft_golden as MS

    for name in ("e2e_sea_raft_iters0", "e2e_sea_raft_l3r3b3"):
        recipe, g = load_golden(name)
        out = MS.reference_e2e(recipe)
        assert np.abs(out["flows"].numpy() - g["flows"]).max() < 1e-5, name
