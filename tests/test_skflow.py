"""CPU: SKFlow.

The oracle's SKFlow stages (tests/skflow_oracle.py) against the reference's own outputs (tests/golden/op_skflow.npz, e2e_skflow_*.npz,
state_shapes_skflow.json, written by tests/make_skflow_golden.py), the model's parameter surface and hyperparameter checks, and the
C header mirrors of the new epilogues, structs and entry points.
"""
import ctypes as C
import json
import os
import re
from argparse import Namespace

import numpy as np
import pytest
import torch

import skflow_oracle as SO
from helpers import GOLDEN, load_golden
from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from ptlflow_b200 import _lib as L
    from ptlflow_b200.csrc import build as B

    if not os.path.exists(L.LIB_PATH):
        B.build()
    return L


def _header() -> str:
    text = open(os.path.join(ROOT, "include", "ptlflow_b200.h")).read()
    return re.sub(r"/\*.*?\*/", " ", text, flags=re.S)


def _forward(recipe):
    sd, img, kw = SO.e2e_inputs(recipe)
    init = None
    if recipe.get("warm"):
        from ptlflow_b200.utils.warm_start import forward_interpolate_batch

        first = SO.raft_forward(sd, img, **kw)
        init = forward_interpolate_batch(first["flow_small"])
    return SO.raft_forward(sd, img, flow_init=init, **kw)


@pytest.mark.parametrize("name", SO.E2E)
def test_skflow_e2e_matches_reference(name):
    recipe, g = load_golden(name)
    out = _forward(recipe)
    assert out["flows"].shape == g["flows"].shape
    assert np.isfinite(g["flows"]).all() and np.abs(g["flows"]).max() > 0.5  # the fixture is not degenerate
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 2e-4
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 2e-4


def test_skflow_warm_start_first_pass():
    recipe, g = load_golden("e2e_skflow_warm")
    sd, img, kw = SO.e2e_inputs(recipe)
    first = SO.raft_forward(sd, img, **kw)
    assert np.abs(first["flow_small"].numpy() - g["first_flow_small"]).max() < 2e-4


@pytest.mark.parametrize("b,h,w", SO.OP_GRIDS)
def test_skflow_operators(b, h, w):
    g = np.load(os.path.join(GOLDEN, "op_skflow.npz"))
    for name, cin, cout, kind in SO.OP_BLOCKS:
        sd, ks, x = SO.op_block_inputs(name, cin, cout, kind, b, h, w)
        out = SO.pc_block(x, sd, "", ks).numpy().reshape(-1)
        assert np.abs(out[SO.op_sample(out.size)] - g[f"{name}_{h}x{w}"]).max() < 1e-5, name
    sd, net, inp, corr, flow, attn = SO.op_iter_inputs(b, h, w)
    for key, arr in zip(("net", "mask", "delta"), SO.update_block(net, inp, corr, flow, attn, sd)):
        flat = arr.numpy().reshape(-1)
        assert np.abs(flat[SO.op_sample(flat.size)] - g[f"iter_{key}_{h}x{w}"]).max() < 1e-5, key


def test_state_dict_contract():
    with open(os.path.join(GOLDEN, "state_shapes_skflow.json")) as f:
        ref = {k: tuple(v) for k, v in json.load(f).items()}
    assert SO.state_dict_shapes() == ref
    import ptlflow_b200 as pb

    m = pb.get_model("skflow")
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == ref
    assert list(m.state_dict().keys()) == list(ref.keys())
    assert "skflow" in pb.get_trainable_model_names()
    assert set(m.pretrained_checkpoints) == {"kitti", "sintel", "things"}


def test_state_dict_variants_load_strictly():
    import ptlflow_b200 as pb

    for kw in (dict(num_heads=2, position_and_content=True), dict(k_conv=(1, 5, 9), PCUpdater_conv=(3,)), dict(corr_levels=3, corr_radius=3)):
        shapes = SO.state_dict_shapes(kw.get("k_conv", (1, 15)), kw.get("PCUpdater_conv", (1, 7)), kw.get("num_heads", 1),
                                      kw.get("corr_levels", 4), kw.get("corr_radius", 4))
        m = pb.get_model("skflow", args=Namespace(model=Namespace(**kw)))
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == shapes
        res = m.load_state_dict(SO.synth_state_dict(shapes, 1), strict=True)
        assert not res.missing_keys and not res.unexpected_keys


@pytest.mark.parametrize("kw", [dict(k_conv=(1, 14)), dict(k_conv=(0,)), dict(k_conv=(33,)), dict(PCUpdater_conv=(2,)),
                                dict(PCUpdater_conv=(-1, 7)), dict(k_conv=(1.0, 15)), dict(k_conv=(1,) * 9)])
def test_kernel_sizes_are_validated(kw):
    import ptlflow_b200 as pb

    with pytest.raises(ValueError, match="odd kernel sizes"):
        pb.get_model("skflow", args=Namespace(model=Namespace(**kw)))


def test_positional_grid_limit_is_checked_on_the_host():
    import ptlflow_b200 as pb

    m = pb.get_model("skflow", args=Namespace(model=Namespace(position_and_content=True)))
    m._check_grid(160, 160)
    with pytest.raises(ValueError, match="160"):
        m._check_grid(161, 20)
    pb.get_model("skflow")._check_grid(161, 300)


def test_header_mirrors():
    """New epilogues, conv-parameter fields, SKFlow structs and block ids of include/ptlflow_b200.h == their ctypes mirrors."""
    L = _lib()
    text = _header()
    body = re.search(r"typedef\s+enum\s*\{([^}]*)\}\s*pfb_epilogue\s*;", text, flags=re.S).group(1)
    vals = dict(re.findall(r"(PFB_EPI_\w+)\s*=\s*(\d+)", body))
    for name in ("GELU", "RESIDUAL_GELU", "LINEAR_APPEND_FLOW", "LINEAR_F32", "AXPY"):
        assert int(vals["PFB_EPI_" + name]) == getattr(L, "EPI_" + name), name
    body = re.search(r"typedef\s+struct\s*\{([^{}]*)\}\s*pfb_conv_params\s*;", text, flags=re.S).group(1)
    fields = re.findall(r"(\w+)\s*(?:\[[^\]]*\])?\s*[;,]", body)
    assert [f[0] for f in L.ConvParams._fields_][-5:] == ["residual", "residual_stride", "residual_offset", "post_w", "post_b"]
    assert fields[-5:] == ["residual", "residual_stride", "residual_offset", "post_w", "post_b"]
    body = re.search(r"typedef\s+enum\s*\{([^}]*)\}\s*pfb_skflow_block_id\s*;", text, flags=re.S).group(1)
    names = [n.split("=")[0].strip() for n in body.split(",") if n.strip()]
    for i, n in enumerate(names):
        assert getattr(L, n[len("PFB_"):]) == i, n
    assert int(re.search(r"#define\s+PFB_SK_MAX_DW\s+(\d+)", text).group(1)) == L.PFB_SK_MAX_DW
    assert int(re.search(r"#define\s+PFB_KERNEL_CLASSES\s+(\d+)", text).group(1)) == L.KERNEL_CLASSES
    for struct, mirror in (("pfb_pc_block", L.PcBlock), ("pfb_skflow_weights", L.SkflowWeights)):
        body = re.search(r"typedef\s+struct\s*\{([^{}]*)\}\s*" + struct + r"\s*;", text, flags=re.S).group(1)
        fields = re.findall(r"(\w+)\s*(?:\[[^\]]*\])?\s*[;,]", body)
        assert fields == [f[0] for f in mirror._fields_], struct
    # the raft loop keeps its layer table and cfg unchanged: skflow has its own weights struct
    assert [f[0] for f in L.RaftCfg._fields_][-1] == "num_heads"
    assert L.L_COUNT == 25


def _cfg(L, variant, **kw):
    a = dict(dtype=L.BF16, B=2, H=16, W=24, feat=256, levels=4, radius=4, iters=4, alt=0, heads=1)
    a.update(kw)
    return L.RaftCfg(variant, a["dtype"], a["B"], a["H"], a["W"], a["feat"], a["levels"], a["radius"], 128, 128, a["iters"], a["alt"],
                     8 * a["H"], 8 * a["W"], 0, 0, 0, 0, 0, a["heads"])


def test_skflow_entry_points_check_their_arguments():
    L = _lib()
    lib = L.load()
    assert lib.pfb_skflow_workspace_bytes(C.byref(_cfg(L, 3))) > 0
    assert lib.pfb_skflow_workspace_bytes(C.byref(_cfg(L, 2))) == 0  # variant 3 only
    assert lib.pfb_raft_workspace_bytes(C.byref(_cfg(L, 3))) == 0  # the raft loop keeps refusing it
    P = 2 * 16 * 24
    big = lib.pfb_skflow_workspace_bytes(C.byref(_cfg(L, 3, heads=4)))
    assert big - lib.pfb_skflow_workspace_bytes(C.byref(_cfg(L, 3))) >= (P * 3 * 128 + P * 4 * 128) * 2
    buf = L.RaftBuffers()
    w = L.SkflowWeights()
    assert lib.pfb_skflow_refine(C.byref(_cfg(L, 3)), C.byref(w), C.byref(buf), None) == -1
    assert lib.pfb_raft_refine(C.byref(_cfg(L, 3)), C.byref(L.RaftWeights()), C.byref(buf), None) == -1
    assert b"variant" in lib.pfb_last_error()


def test_depthwise_argument_checks():
    L = _lib()
    lib = L.load()
    # even kernel, k > 31, odd channel count, odd offset
    assert lib.pfb_depthwise_conv_gelu(16, 64, 0, 16, 64, 0, 16, 16, 1, 8, 8, 64, 4, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_gelu(16, 64, 0, 16, 64, 0, 16, 16, 1, 8, 8, 64, 33, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_gelu(16, 64, 0, 16, 64, 0, 16, 16, 1, 8, 8, 63, 3, L.BF16, None) == -1
    assert lib.pfb_depthwise_conv_gelu(16, 64, 1, 16, 64, 0, 16, 16, 1, 8, 8, 62, 3, L.BF16, None) == -1


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout absent")
def test_live_reference_agrees_with_skflow_fixtures():
    """Where the reference checkout exists, re-run the real reference for the SKFlow fixtures: they are not stale."""
    import make_skflow_golden as MS

    g = np.load(os.path.join(GOLDEN, "op_skflow.npz"))
    b, h, w = SO.OP_GRIDS[0]
    for name, cin, cout, kind in SO.OP_BLOCKS:
        out = MS.reference_block(name, cin, cout, kind, b, h, w).reshape(-1)
        assert np.array_equal(out[SO.op_sample(out.size)], g[f"{name}_{h}x{w}"]), name
    for name in ("e2e_skflow_default", "e2e_skflow_kconv"):
        recipe, gg = load_golden(name)
        out, _ = MS.reference_e2e(recipe)
        assert np.abs(out["flows"].numpy() - gg["flows"]).max() < 1e-5, name
