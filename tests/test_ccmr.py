"""CPU: CCMR / CCMR+ -- the fp32 oracle against the reference's fixtures, the state-dict contract, the host checks and the C-ABI
argument checks of the a18 entry points."""
import ctypes as C
import json
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import ccmr_oracle as CC  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


def _lib():
    from ptlflow_b200 import _lib as L
    from ptlflow_b200.csrc import build as B

    if not os.path.exists(L.LIB_PATH):
        B.build()
    return L


@pytest.mark.parametrize("name", CC.E2E)
def test_ccmr_e2e_oracle_matches_reference(name):
    case = CC.E2E_CASES[CC.E2E.index(name)]
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    rec = CC.recipe_of(case)
    assert json.loads(g["recipe"].tobytes()) == json.loads(json.dumps(rec))
    fi = torch.from_numpy(g["flow_init"]) if rec["warm"] else None
    out = CC.forward_recipe(rec, fi)
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 2e-4
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 2e-4


def test_ccmr_operators():
    g = np.load(os.path.join(GOLDEN, "op_ccmr.npz"))
    sd, x = CC.op_inputs()
    with torch.no_grad():
        np.testing.assert_allclose(CC.xcit(sd, "xcit.1.", x["ctx"]).numpy(), g["xcit_self"], atol=2e-4)
        np.testing.assert_allclose(CC.xcit(sd, "update_block.aggregator.1.", x["gc"], x["ctx"]).numpy(), g["xcit_agg"], atol=2e-4)
        net, mask, delta = CC.update_block(x["net"], x["inp"], x["corr"], x["flow"], x["gc"], sd, 1)
        grid = CC.O.coords_grid(2, 12, 18)
        hand = grid + CC.MS.convex_up2(x["coords"] - CC.O.coords_grid(2, 6, 9), x["mask"])
        up2 = CC.upflow2(x["flow_lo"])
    for k, v in dict(net=net, mask=mask, delta=delta, handover=hand, upflow2=up2).items():
        np.testing.assert_allclose(v.numpy(), g[k], atol=2e-4, err_msg=k)


@pytest.mark.parametrize("model", ["ccmr", "ccmr_p"])
def test_state_dict_contract(model):
    import ptlflow_b200 as pb

    m = pb.get_model(model)
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == CC.state_dict_shapes(model)
    assert not any("refine" in k.lower() for k in mine)  # RefineHead is defined by the reference but never instantiated
    m.load_state_dict(CC.synth_state_dict(CC.state_dict_shapes(model), 1), strict=True)


def test_checkpoint_loads_offline(tmp_path):
    import ptlflow_b200 as pb

    sd = CC.synth_state_dict(CC.state_dict_shapes("ccmr_p"), 3)
    path = tmp_path / "ccmr_p.ckpt"
    torch.save({"state_dict": sd}, path)
    m = pb.get_model("ccmr_p", ckpt_path=str(path))
    assert torch.equal(m.state_dict()["xcit.0.blocks.0.gamma1"], sd["xcit.0.blocks.0.gamma1"])


def test_registry_and_defaults():
    import ptlflow_b200 as pb
    from ptlflow_b200 import get_trainable_model_names

    assert {"ccmr", "ccmr_p"} <= set(get_trainable_model_names())
    a, b = pb.get_model("ccmr"), pb.get_model("ccmr_p")
    assert a.iters == (8, 10, 15) and b.iters == (8, 10, 10, 10)
    assert (a.num_scales, b.num_scales) == (3, 4) and a.model_type == "CCMR" and b.model_type == "CCMR+"
    assert a.output_stride == b.output_stride == 32 and a.alternate_corr and a.lookup_pyramid_levels == 2 and a.lookup_radius == 4
    assert set(a.pretrained_checkpoints) == set(b.pretrained_checkpoints) == {"kitti", "sintel"}


@pytest.mark.parametrize("model,iters", [("ccmr", (8, 10)), ("ccmr", (8, 10, 15, 2)), ("ccmr_p", (8, 10, 15)), ("ccmr_p", (1, 0, 1, 1)),
                                         ("ccmr", 7)])
def test_bad_iters_raise(model, iters):
    import ptlflow_b200 as pb

    with pytest.raises(ValueError, match="iters"):
        pb.get_model(model, args=Namespace(model=Namespace(iters=iters)))
    m = pb.get_model(model)
    m.iters = iters
    with pytest.raises(ValueError, match="iters"):
        m._check_grid(2, 3)


@pytest.mark.parametrize("kw,match", [(dict(model_type="CCMR+"), "num_scales"), (dict(num_scales=4), "num_scales"),
                                      (dict(cnet_norm="batch"), "out of scope"), (dict(fnet_norm="instance"), "out of scope")])
def test_unsupported_configurations_raise(kw, match):
    import ptlflow_b200 as pb

    with pytest.raises(ValueError, match=match):
        pb.get_model("ccmr", args=Namespace(model=Namespace(**kw)))


def test_grid_warm_start_and_volume_checks_on_the_host():
    import ptlflow_b200 as pb

    m = pb.get_model("ccmr")
    m._check_grid(1, 1)  # a 2x2 grid at 1/16 holds the 2 lookup levels
    with pytest.raises(ValueError, match="lookup_pyramid_levels"):
        pb.get_model("ccmr", args=Namespace(model=Namespace(lookup_pyramid_levels=3)))._check_grid(1, 4)
    # stride-32 padding: a warm start on sizes that are not multiples of 32 fails in the reference, and here before any launch
    with pytest.raises(ValueError, match="multiples of 32"):
        m({"images": torch.zeros(1, 2, 3, 80, 96), "prev_preds": {"flow_small": torch.zeros(1, 2, 5, 6)}})
    with pytest.raises(RuntimeError, match="CUDA"):
        m({"images": torch.zeros(1, 2, 3, 64, 96), "prev_preds": {"flow_small": torch.zeros(1, 2, 4, 6)}})
    v = pb.get_model("ccmr_p", args=Namespace(model=Namespace(alternate_corr=False)))
    with pytest.raises(ValueError, match="alternate_corr=True"):
        v._check_volume(torch.zeros(1, 2, 3, 436, 1024))
    v._check_volume(torch.zeros(1, 2, 3, 64, 96))


def _cfg(L, variant, **kw):
    a = dict(dtype=L.BF16, B=2, H=16, W=24, feat=128, levels=2, radius=4, iters=4, alt=1)
    a.update(kw)
    return L.RaftCfg(variant, a["dtype"], a["B"], a["H"], a["W"], a["feat"], a["levels"], a["radius"], 128, 128, a["iters"], a["alt"],
                     2 * a["H"], 2 * a["W"], 0, 0, 0, 0, 0, 1)


def test_ccmr_entry_points_check_their_arguments():
    L = _lib()
    lib = L.load()
    n6 = lib.pfb_ccmr_workspace_bytes(C.byref(_cfg(L, 6)))
    assert n6 > lib.pfb_msraft_workspace_bytes(C.byref(_cfg(L, 5))) > 0
    assert lib.pfb_ccmr_workspace_bytes(C.byref(_cfg(L, 5))) == 0  # variant 6 only
    for fn in (lib.pfb_raft_workspace_bytes, lib.pfb_msraft_workspace_bytes, lib.pfb_skflow_workspace_bytes, lib.pfb_searaft_workspace_bytes):
        assert fn(C.byref(_cfg(L, 6))) == 0  # every other loop refuses it
    buf, w = L.RaftBuffers(), L.CcmrWeights()
    assert lib.pfb_ccmr_refine(C.byref(_cfg(L, 5)), C.byref(w), C.byref(buf), 0.0, 0, None, None) == -1
    assert b"variant" in lib.pfb_last_error()
    assert lib.pfb_ccmr_refine(C.byref(_cfg(L, 6)), None, C.byref(buf), 0.0, 0, None, None) == -1
    assert lib.pfb_ccmr_update_iter(C.byref(_cfg(L, 0)), C.byref(w), C.byref(buf), None, None, 0.0, None) == -1
    assert lib.pfb_xcit_context(C.byref(_cfg(L, 6)), C.byref(w), 16, 16, 16, 16, None) == -1  # workspace too small
    assert b"workspace" in lib.pfb_last_error()
    assert lib.pfb_msraft_refine(C.byref(_cfg(L, 6)), C.byref(w.raft), C.byref(buf), 0.0, None, None) == -1


def test_new_kernels_check_their_arguments():
    L = _lib()
    lib = L.load()
    assert lib.pfb_layernorm(None, 128, 0, 16, 128, 0, None, None, 4, 128, 1e-6, L.F16, None) == -1
    assert lib.pfb_layernorm(16, 128, 0, 16, 128, 0, 16, None, 4, 128, 1e-6, L.F16, None) == -1  # gamma without beta
    assert lib.pfb_layernorm(16, 128, 0, 16, 128, 0, None, None, 4, 1024, 1e-6, L.F16, None) == -1  # C > 512
    assert lib.pfb_depthwise_conv3x3_ex(16, 128, 0, 16, 128, 0, 16, 16, None, 0, 0, 1, 4, 4, 128, 2, L.F16, None) == -1  # mode
    assert lib.pfb_depthwise_conv3x3_ex(16, 128, 0, 16, 128, 0, 16, 16, None, 0, 0, 1, 4, 4, 128, 1, L.F16, None) == -1  # no addend
    assert lib.pfb_fourier_features(16, 0, 4, L.F16, None) == -1
    assert lib.pfb_xca_stats(16, 200, 0, 128, 1, 64, 16, 16, L.F16, None) == -1  # k columns outside the row
    assert lib.pfb_xca_stats_workspace_bytes(1, 513) == 2 * 2304 * 4
    assert lib.pfb_xca_fold(16, None, 16, 16, 16, 16, 16, None, 16, 1, L.F16, None) == -1
    assert lib.pfb_upflow2(16, 16, 1, 4, 4, 8, 8, 1, 0, None) == -1  # window outside the 2x grid
    assert lib.pfb_convex_handover2x(None, 16, 16, 1, 4, 4, L.F16, None) == -1
    assert lib.pfb_convex_upsample2x(16, 16, 16, 2, 1, 4, 4, 8, 8, 0, 0, L.F16, None) == -1  # modes 0 and 1 only
