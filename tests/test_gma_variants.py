"""CPU: GMA's position-only, position-and-content and multi-head attention.

The oracle's GMA-variant stages (tests/gma_oracle.py) against the reference's own outputs for these variants (tests/golden/op_gma_variants.npz,
e2e_gma_*.npz, state_shapes_gma_heads4.json, written by tests/make_gma_golden.py), the model's parameter surface, the grid limit
of the positional modes and the C header mirrors of the new configuration field and layer id.
"""
import json
import os
import re
from argparse import Namespace

import numpy as np
import pytest
import torch

import gma_oracle as GO
from helpers import GOLDEN, load_golden
from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle_variant(mode, heads, b, h, w):
    """(attention [b, heads, N, N], aggregate [b, 128, h, w]) of the oracle for one op_gma_variants case."""
    sd, inp, motion = GO.op_inputs(heads, b, h, w)
    attn = GO.attention(inp, sd, heads, **GO.MODES[mode])
    return attn, GO.aggregate(attn, motion, sd)


@pytest.mark.parametrize("name", GO.E2E)
def test_gma_variant_e2e_matches_reference(name):
    recipe, g = load_golden(name)
    sd, img, kw = GO.e2e_inputs(recipe)
    out = GO.raft_forward(sd, img, **kw)
    assert out["flows"].shape == g["flows"].shape
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 2e-4
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 2e-4


@pytest.mark.parametrize("mode,heads,b,h,w", GO.OP_CASES, ids=[f"{m}-h{k}-{hh}x{ww}" for m, k, _, hh, ww in GO.OP_CASES])
def test_gma_variant_attention_and_aggregate(mode, heads, b, h, w):
    g = np.load(os.path.join(GOLDEN, "op_gma_variants.npz"))
    key = f"{mode}_h{heads}_{h}x{w}"
    attn, agg = oracle_variant(mode, heads, b, h, w)
    assert tuple(attn.shape) == tuple(g[key + "_attention_shape"])
    assert tuple(agg.shape) == tuple(g[key + "_aggregate_shape"])
    assert (attn.sum(-1) - 1).abs().max().item() < 1e-5
    for name, mine, tol in (("attention", attn, 1e-6), ("aggregate", agg, 2e-5)):
        flat = mine.numpy().reshape(-1)
        assert np.abs(flat[GO.op_sample(flat.size)] - g[f"{key}_{name}"]).max() < tol, name


def test_positional_logits_are_not_negligible():
    """The synthetic rel_height / rel_width tables have nn.Embedding's N(0, 1) scale: the positional logits are O(1), so a
    transposed or shifted table index changes the attention far beyond any tolerance."""
    sd, inp, _ = GO.op_inputs(1, 2, 6, 9)
    attn = GO.attention(inp, sd, position_only=True)
    q = torch.nn.functional.conv2d(inp, sd["att.to_qk.weight"])[:, :128].reshape(2, 1, 128, 6, 9) * 128 ** -0.5
    assert GO.position_logits(q, sd).std().item() > 0.3
    swapped = dict(sd)
    swapped["att.pos_emb.rel_height.weight"], swapped["att.pos_emb.rel_width.weight"] = sd["att.pos_emb.rel_width.weight"], sd["att.pos_emb.rel_height.weight"]
    assert (GO.attention(inp, swapped, position_only=True) - attn).abs().max().item() > 1e-2


def test_position_only_wins_over_position_and_content():
    sd, inp, _ = GO.op_inputs(2, 1, 6, 9)
    both = GO.attention(inp, sd, 2, position_only=True, position_and_content=True)
    assert torch.equal(both, GO.attention(inp, sd, 2, position_only=True))


def test_state_dict_contract_heads4():
    with open(os.path.join(GOLDEN, "state_shapes_gma_heads4.json")) as f:
        ref = {k: tuple(v) for k, v in json.load(f).items()}
    assert GO.state_dict_shapes(4) == ref
    import ptlflow_b200 as pb

    m = pb.get_model("gma", args=Namespace(model=Namespace(num_heads=4)))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == ref


def test_positional_grid_limit_is_checked_on_the_host():
    """The position tables cover offsets below max_pos_size = 160: larger grids are refused with a ValueError (the check runs
    before anything is launched); content attention has no such limit."""
    import ptlflow_b200 as pb

    for flags in ({"position_only": True}, {"position_and_content": True}, {"position_and_content": True, "num_heads": 2}):
        m = pb.get_model("gma", args=Namespace(model=Namespace(**flags)))
        m._check_grid(160, 160)
        with pytest.raises(ValueError, match="160"):
            m._check_grid(161, 20)
        with pytest.raises(ValueError, match="160"):
            m._check_grid(20, 200)
    pb.get_model("gma")._check_grid(161, 300)


def test_layer_ids_mirror_the_header():
    """pfb_layer_id of include/ptlflow_b200.h (incl. PFB_L_AGG_PROJ) == the L_* constants of ptlflow_b200/_lib.py."""
    from ptlflow_b200 import _lib

    text = open(os.path.join(ROOT, "include", "ptlflow_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    body = re.search(r"typedef\s+enum\s*\{([^}]*)\}\s*pfb_layer_id\s*;", text, flags=re.S).group(1)
    names = [n.split("=")[0].strip() for n in body.split(",") if n.strip()]
    assert names[-2:] == ["PFB_L_AGG_PROJ", "PFB_L_COUNT"]
    for i, n in enumerate(names):
        assert getattr(_lib, n[len("PFB_"):]) == i, n
    assert [f[0] for f in _lib.RaftCfg._fields_][-1] == "num_heads"


def test_workspace_grows_with_heads():
    import ctypes as C

    from ptlflow_b200 import _lib
    from ptlflow_b200.csrc import build as B

    if not os.path.exists(_lib.LIB_PATH):
        B.build()
    lib = _lib.load()
    sizes = []
    for heads in (0, 1, 4):
        cfg = _lib.RaftCfg(_lib.VARIANT_GMA, _lib.BF16, 4, 55, 128, 256, 4, 4, 128, 128, 12, 0, 436, 1024, 2, 0, 0, 1, 0, heads)
        sizes.append(lib.pfb_raft_workspace_bytes(C.byref(cfg)))
    assert sizes[0] == sizes[1] > 0
    P, N = 4 * 55 * 128, 55 * 128
    # v and its transpose for 3 more heads, and the concatenated per-head outputs of 4 heads
    assert sizes[2] - sizes[1] >= (P * 3 * 128 + 4 * 3 * 128 * N + P * 4 * 128) * 2
    bad = _lib.RaftCfg(_lib.VARIANT_RAFT, _lib.BF16, 1, 16, 32, 256, 4, 4, 128, 128, 4, 0, 128, 256, 0, 0, 0, 0, 0, 2)  # heads on raft
    assert lib.pfb_raft_workspace_bytes(C.byref(bad)) == 0


def test_relpos_softmax_argument_checks():
    from ptlflow_b200 import _lib
    from ptlflow_b200.csrc import build as B

    if not os.path.exists(_lib.LIB_PATH):
        B.build()
    lib = _lib.load()
    # grid beyond the table, table stride too short, rows not a multiple of H*W
    assert lib.pfb_attention_softmax_relpos(None, 16, 16, 319, 16, 161 * 4, 161, 4, 160, 1, None) == -1
    assert b"position table" in lib.pfb_last_error()
    assert lib.pfb_attention_softmax_relpos(None, 16, 16, 300, 16, 64, 8, 8, 160, 1, None) == -1
    assert lib.pfb_attention_softmax_relpos(None, 16, 16, 319, 16, 65, 8, 8, 160, 1, None) == -1
    assert lib.pfb_attention_softmax_relpos(None, None, 16, 319, 16, 64, 8, 8, 160, 1, None) == -1


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout absent")
def test_live_reference_agrees_with_gma_variant_fixtures():
    """Where the reference checkout exists, re-run the real reference for the GMA-variant fixtures: they are not stale."""
    import make_gma_golden as MG

    g = np.load(os.path.join(GOLDEN, "op_gma_variants.npz"))
    for mode, heads, b, h, w in GO.OP_CASES:
        key = f"{mode}_h{heads}_{h}x{w}"
        a, agg = MG.reference_op_outputs(mode, heads, b, h, w)
        for name, arr in (("attention", a), ("aggregate", agg)):
            flat = arr.reshape(-1)
            assert np.array_equal(flat[GO.op_sample(flat.size)], g[f"{key}_{name}"]), key
    for name in GO.E2E:
        recipe, gg = load_golden(name)
        out = MG.reference_e2e(recipe)
        assert np.abs(out["flows"].numpy() - gg["flows"]).max() < 1e-5, name
