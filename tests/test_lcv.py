"""CPU: LCV -- the fp32 oracle against the reference's fixtures (and the live reference where its checkout exists), the state-dict and
hparams contract, the level sizes of pfb_corr_level_sizes, and the argument checks of pfb_corr_lookup_tiled_ex without a launch."""
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
import lcv_oracle as LO  # noqa: E402
from oracle import ref_shim  # noqa: E402
from helpers import check_live_reference, check_oracle_fixture, lib as _lib  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


@pytest.mark.parametrize("name", LO.E2E)
def test_lcv_e2e_oracle_matches_reference(name):
    check_oracle_fixture(LO, name, 2e-4, 2e-4)


def test_lcv_operators():
    g = np.load(os.path.join(GOLDEN, "op_lcv.npz"))
    with LO.O.fp32_strict(), torch.no_grad():
        out = LO.op_outputs()
    np.testing.assert_allclose(out["W"].numpy(), g["W"], atol=1e-5, rtol=0)
    np.testing.assert_array_equal(out["level_sizes"].numpy(), g["level_sizes"])
    assert g["level_sizes"].tolist() == [[12, 13], [6, 6], [6, 6], [6, 6]]
    np.testing.assert_allclose(out["lookup"].numpy(), g["lookup"], atol=1e-4, rtol=0)
    # the recipe's W is symmetric positive definite and far from the identity of the reference's initialisation
    W = torch.from_numpy(g["W"]).double()
    assert torch.allclose(W, W.t(), atol=1e-5) and torch.linalg.eigvalsh((W + W.t()) / 2).min() > 0
    assert (W - torch.eye(W.shape[0], dtype=W.dtype)).abs().max() > 0.5


@pytest.mark.skipif(not ref_shim.available(), reason="the reference checkout is not available")
def test_lcv_fixtures_match_live_reference():
    import make_lcv_golden as MK

    check_live_reference(MK, LO, ["e2e_lcv_raft_tiny", "e2e_lcv_raft_small_default"], 2e-4, "op_lcv")


@pytest.mark.parametrize("name,extra", [("lcv_raft", 3), ("lcv_raft_small", 3)])
def test_state_dict_and_hparams(name, extra):
    import ptlflow_b200 as pb

    m = pb.get_model(name)
    sd = m.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == LO.state_dict_shapes(name)
    raft = pb.get_model(name[len("lcv_"):]).state_dict()
    assert set(sd) - set(raft) == {"corr_block.raw_P", "corr_block.raw_D", "corr_block.eye"} and len(sd) == len(raft) + extra
    m.load_state_dict(LO.synth_state_dict(name, 1), strict=True)
    hp = vars(m.hparams)
    assert "alternate_corr" not in hp
    assert {k: hp[k] for k in ("corr_levels", "corr_radius", "dropout", "gamma", "max_flow", "iters")} == dict(
        corr_levels=4, corr_radius=4 if name == "lcv_raft" else 3, dropout=0.0, gamma=0.8, max_flow=400, iters=32)
    assert set(m.pretrained_checkpoints) == ({"chairs", "things"} if name == "lcv_raft" else set())
    with pytest.raises(TypeError, match="alternate_corr"):
        type(m)(alternate_corr=True)


# (H, W, levels, pool_min_side) -> level sizes, distinct levels
LEVEL_TABLE = [
    ((17, 21, 4, 0), [(17, 21), (8, 10), (4, 5), (2, 2)], 4),  # RAFT's rule
    ((4, 4, 4, 0), [(4, 4), (2, 2), (1, 1), (0, 0)], 4),  # RAFT's pyramid of a 4x4 grid has an empty level
    ((17, 21, 4, 9), [(17, 21), (8, 10), (8, 10), (8, 10)], 2),  # LCV r=4
    ((8, 8, 4, 9), [(8, 8)] * 4, 1),
    ((4, 4, 4, 9), [(4, 4)] * 4, 1),
    ((40, 48, 4, 9), [(40, 48), (20, 24), (10, 12), (5, 6)], 4),  # every level pools from 40 px per side
    ((39, 48, 4, 9), [(39, 48), (19, 24), (9, 12), (9, 12)], 3),
    ((55, 128, 4, 9), [(55, 128), (27, 64), (13, 32), (6, 16)], 4),
    ((16, 20, 3, 7), [(16, 20), (8, 10), (4, 5)], 3),  # LCV r=3, L=3
    ((12, 16, 4, 7), [(12, 16), (6, 8), (6, 8), (6, 8)], 2),
]


@pytest.mark.parametrize("args,sizes,distinct", LEVEL_TABLE)
def test_level_sizes(args, sizes, distinct):
    _lib()
    from ptlflow_b200 import ops

    assert ops.corr_level_sizes(*args) == (sizes, distinct)
    H, W, L, m = args
    if m:
        assert LO.level_sizes(H, W, L, (m - 1) // 2) == sizes


def test_argument_checks_without_a_launch():
    L = _lib()
    lib = L.load()
    lh, lw = (C.c_int * 4)(), (C.c_int * 4)()
    for bad in ((0, 4, 4, 0), (4, 4, 0, 0), (4, 4, 9, 0), (4, 4, 4, -1)):
        assert lib.pfb_corr_level_sizes(*bad, lh, lw) == -1, bad
    assert lib.pfb_corr_level_sizes(4, 4, 4, 9, None, lw) == -1
    n0 = lib.pfb_launch_count(-1)
    dummy = (C.c_void_p * 4)(*([16] * 4))
    pp = C.cast(dummy, C.POINTER(C.c_void_p))
    sizes_h, sizes_w = (C.c_int * 4)(8, 8, 8, 8), (C.c_int * 4)(10, 10, 10, 10)
    ok = dict(B=1, H=8, W=10, H2=8, W2=10, levels=4, radius=4, dtype=L.F16, stride=328)

    def call(lh_, lw_, **kw):
        a = {**ok, **kw}
        return lib.pfb_corr_lookup_tiled_ex(pp, lh_, lw_, 16, 16, a["B"], a["H"], a["W"], a["H2"], a["W2"], a["levels"], a["radius"],
                                            a["dtype"], a["stride"], None)

    assert call(sizes_h, None) == -1 and b"come together" in lib.pfb_last_error()
    assert call(sizes_h, sizes_w, dtype=L.F32) == -1
    assert call(sizes_h, sizes_w, levels=5) == -1
    assert call(sizes_h, sizes_w, stride=320) == -1
    assert call((C.c_int * 4)(8, 8, 0, 8), sizes_w) == -1 and b"empty" in lib.pfb_last_error()
    assert call(sizes_h, sizes_w, radius=5, stride=488) == -3  # PFB_ERR_UNSUPPORTED: no kernel for radius 5
    assert lib.pfb_launch_count(-1) == n0
    # a 4x4 grid with 4 levels: RAFT's pyramid has an empty level, LCV's (pool_min_side 9) does not
    cfg = L.RaftCfg(0, L.F16, 1, 4, 4, 0, 4, 4, 128, 128, 2, 0, 32, 32, 0, 0, 0)
    assert lib.pfb_raft_workspace_bytes(C.byref(cfg)) == 0 and lib.pfb_raft_workspace_bytes_ex(C.byref(cfg), 0) == 0
    assert lib.pfb_raft_workspace_bytes_ex(C.byref(cfg), 9) > 0 and lib.pfb_raft_workspace_bytes_ex(C.byref(cfg), -1) == 0
    assert L.RaftBuffers._fields_[-1][0] == "pool_min_side"
