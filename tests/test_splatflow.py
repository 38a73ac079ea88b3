"""CPU: SplatFlow.

The oracle (tests/splatflow_oracle.py) against the reference's own outputs (tests/golden/op_splatflow.npz, e2e_splatflow_*.npz,
state_shapes_splatflow.json, written by tests/make_splatflow_golden.py) and against the live reference where its checkout exists;
the splat stand-in of the generator against a brute-force float64 loop; the model's parameter surface; the host-only checks of
the loop's cfg (context 256) and of the motion-buffer query.
"""
import ctypes as C
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

import ptlflow_b200 as pb  # (before any reference import: oracle.ref_shim stands in a LightningModule of its own)
import splatflow_oracle as SO
from helpers import GOLDEN, check_live_reference, check_oracle_fixture, lib as _lib, load_golden, load_golden_arrays, raft_cfg
from oracle import ref_shim

TOL = 2e-4


@pytest.mark.parametrize("name", SO.E2E)
def test_oracle_matches_reference_fixtures(name):
    g = check_oracle_fixture(SO, name, TOL)
    assert np.isfinite(g["flows"]).all() and np.abs(g["flows"]).max() > 0.5  # the fixture is not degenerate


def test_fixture_cases_differ_where_they_should():
    """Three frames change the output (mf_t is live), and the prev_preds / corr_radius cases equal a plain three-frame run."""
    rec3 = SO.recipe_of(SO.E2E_CASES[SO.E2E.index("e2e_splatflow_three")])
    two = SO.forward_recipe({**rec3, "frames": 2})["flows"]
    assert np.abs(two.numpy() - load_golden("e2e_splatflow_three")[1]["flows"]).max() > 0.1
    for name in ("e2e_splatflow_prev", "e2e_splatflow_r3"):
        rec = SO.recipe_of(SO.E2E_CASES[SO.E2E.index(name)])
        plain = SO.forward_recipe({**rec, "kwargs": {"iters": rec["kwargs"]["iters"]}, "prev": False})
        assert np.abs(plain["flows"].numpy() - load_golden(name)[1]["flows"]).max() < TOL, name


def test_operators_match_reference():
    g = load_golden_arrays("op_splatflow")
    x, flow = SO.op_splat_inputs()
    np.testing.assert_allclose(SO.softsplat_average(x, flow).numpy(), g["splat"], atol=0, rtol=0)
    sd, net, inp, corr, flow, attn, mf_t = SO.op_iter_inputs()
    n, m, d, mf = SO.update(net, inp, corr, flow, attn, SO._as_gma(sd, True), mf_t)
    for key, v in (("net", n), ("mask", m), ("delta", d), ("mf", mf)):
        np.testing.assert_allclose(v.numpy(), g["iter_" + key], atol=2e-5, rtol=0, err_msg=key)


def test_splat_stand_in_against_float64_loop():
    """The generator's restatement of the cupy kernel and the oracle's splat equal each other bit for bit, and the float64 loop to
    fp32 rounding; the crafted flows reach every case (out of the image, collisions, empty pixels)."""
    if not ref_shim.available():
        pytest.skip("reference checkout not available")
    import make_splatflow_golden as M

    x, flow = SO.op_splat_inputs()
    a, b, ref = M.softsplat_stand_in(x, flow), SO.softsplat_average(x, flow), SO.softsplat_average_f64(x, flow)
    assert torch.equal(a, b)
    assert (a.double() - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())
    assert ((a == 0).all(dim=1)).any()  # a pixel that receives nothing


def test_live_reference_matches_fixtures():
    if not ref_shim.available():
        pytest.skip("reference checkout not available")
    import make_splatflow_golden as M

    check_live_reference(M, SO, ["e2e_splatflow_two", "e2e_splatflow_three_ragged"], 1e-5, op_fixture="op_splatflow")


def test_state_dict_names_and_shapes():
    want = json.load(open(os.path.join(GOLDEN, "state_shapes_splatflow.json")))
    model = pb.get_model("splatflow", args=Namespace(model=Namespace()))
    got = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert list(got) == list(want) and got == want
    assert {k: list(v) for k, v in SO.state_dict_shapes().items()} == want
    assert model.pretrained_checkpoints == {
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/splatflow-kitti-2aa8e145.ckpt"}


def test_keywords_are_kept_and_the_loop_is_fixed():
    model = pb.get_model("splatflow", args=Namespace(model=Namespace(corr_levels=3, corr_radius=3, alternate_corr=True, iters=7)))
    assert (model.hparams.corr_levels, model.hparams.corr_radius, model.hparams.alternate_corr, model.hparams.iters) == (3, 3, True, 7)
    assert (model.corr_levels, model.corr_radius, model.alternate_corr, model.iters) == (4, 4, False, 7)


def test_fewer_than_two_frames_raise():
    model = pb.get_model("splatflow", args=Namespace(model=Namespace()))
    for shape in ((1, 1, 3, 64, 64), (1, 3, 64, 64)):
        with pytest.raises(ValueError, match="T >= 2"):
            model({"images": torch.zeros(shape)})


GMA_CFG = dict(variant=2, dtype=1, B=2, H=12, W=16, corr_levels=4, corr_radius=4, hidden_dim=128, context_dim=128, iters=1,
               out_h=96, out_w=128)


def test_context_256_is_gma_only():
    L = _lib()
    lib = L.load()
    gma256 = lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, GMA_CFG, context_dim=256)))
    assert gma256 > 0 and gma256 == lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, GMA_CFG)))  # the plan does not read it
    for dtype in (0, 1, 2):
        assert lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, GMA_CFG, context_dim=256, dtype=dtype))) > 0
    for variant in (0, 7, 8):  # raft, flow1d, csflow
        assert lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, GMA_CFG, variant=variant, context_dim=256))) == 0
    assert lib.pfb_raft_workspace_bytes(C.byref(raft_cfg(L, GMA_CFG, context_dim=192))) == 0
    assert lib.pfb_msraft_workspace_bytes(C.byref(raft_cfg(L, GMA_CFG, variant=5, context_dim=256))) == 0


@pytest.mark.parametrize("dtype,es", [(0, 4), (1, 2), (2, 2)])
def test_motion_buffer_query(dtype, es):
    L = _lib()
    lib = L.load()
    off, stride = C.c_size_t(), C.c_int()
    for cd in (128, 256):
        cfg = raft_cfg(L, GMA_CFG, dtype=dtype, context_dim=cd)
        assert lib.pfb_raft_workspace_motion(C.byref(cfg), C.byref(off), C.byref(stride)) == 0
        total = lib.pfb_raft_workspace_bytes(C.byref(cfg))
        P = cfg.B * cfg.H * cfg.W
        assert stride.value == 256 and off.value % 256 == 0 and off.value + P * stride.value * es <= total
    cfg = raft_cfg(L, GMA_CFG, variant=0)
    assert lib.pfb_raft_workspace_motion(C.byref(cfg), C.byref(off), C.byref(stride)) == 0 and stride.value == 128
    assert lib.pfb_raft_workspace_motion(C.byref(raft_cfg(L, GMA_CFG, variant=0, context_dim=256)), C.byref(off), C.byref(stride)) != 0
    assert lib.pfb_raft_workspace_motion(None, C.byref(off), C.byref(stride)) != 0


def test_splat_argument_checks():
    L = _lib()
    lib = L.load()
    assert lib.pfb_softsplat_workspace_bytes(2, 7, 9, 128) == -(-2 * 7 * 9 * 129 * 8 // 256) * 256
    assert lib.pfb_softsplat_workspace_bytes(0, 7, 9, 128) == 0
    p = C.c_void_p(256)
    args = dict(src=p, ss=256, so=0, flow=p, dst=p, ds=256, do=128, ws=p, wsb=1 << 30, B=1, H=4, W=4, C=128, dt=1)
    def call(**kw):
        a = {**args, **kw}
        return lib.pfb_softsplat_average(*a.values(), None)
    assert call(src=None) != 0 and call(ss=100) != 0 and call(do=200) != 0 and call(wsb=16) != 0 and call(C=0) != 0 and call(dt=7) != 0
    assert "softsplat_average" in lib.pfb_last_error().decode()
