"""CPU: LLA-Flow -- the fp32 oracle against the reference's fixtures (and the live reference where its checkout exists), the state-dict
contract, the registry, defaults and hparams, the ``gamma`` name clash, the constructor and grid checks, the one-GEMM form of the volume
in float64, and the C-ABI argument checks of the a22 entry points."""
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

import ptlflow_b200  # noqa: E402,F401  (imported before the reference's shim stubs lightning, so the models keep their hparams)
import llaflow_oracle as LL  # noqa: E402
from oracle import ref_shim  # noqa: E402
from helpers import lib as _lib  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


@pytest.mark.parametrize("name", LL.E2E)
def test_llaflow_e2e_oracle_matches_reference(name):
    case = LL.E2E_CASES[LL.E2E.index(name)]
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    rec = LL.recipe_of(case)
    assert json.loads(g["recipe"].tobytes()) == json.loads(json.dumps(rec))
    fi = torch.from_numpy(g["flow_init"]) if rec["warm"] else None
    out = LL.forward_recipe(rec, fi)
    assert np.abs(out["flows"].numpy() - g["flows"]).max() < 1e-4
    assert np.abs(out["flow_small"].numpy() - g["flow_small"]).max() < 1e-4
    if rec["warm"]:
        first = LL.forward_recipe(rec)
        assert np.abs(first["flow_small"].numpy() - g["prev_flow_small"]).max() < 1e-4


def test_llaflow_operators():
    g = np.load(os.path.join(GOLDEN, "op_llaflow.npz"))
    sd, x = LL.op_inputs()
    with LL.O.fp32_strict(), torch.no_grad():
        out = LL.op_outputs(sd, x)
    for k, v in out.items():
        np.testing.assert_allclose(v.numpy(), g[k], atol=2e-5, rtol=1e-5, err_msg=k)
    np.testing.assert_allclose(g["a1"].sum(-1), 1.0, atol=1e-6)


@pytest.mark.parametrize("name", ["op_llaflow"] + LL.E2E)
def test_fixtures_exercise_the_shift_term(name):
    """Both gammas are 0 at the reference's initialisation; in the fixtures the gamma corr2 term is at least 10 % of the plain term."""
    assert float(np.load(os.path.join(GOLDEN, name + ".npz"))["extra_ratio"]) >= 0.1


@pytest.mark.skipif(not ref_shim.available(), reason="the reference checkout is not available")
def test_llaflow_fixtures_match_live_reference():
    import make_llaflow_golden as MK

    g = np.load(os.path.join(GOLDEN, "op_llaflow.npz"))
    for k, v in MK.reference_ops().items():
        np.testing.assert_allclose(v, g[k], atol=1e-6, rtol=0, err_msg=k)
    for name in ("e2e_llaflow_ragged", "e2e_llaflow_raft_r3"):
        rec = LL.recipe_of(LL.E2E_CASES[LL.E2E.index(name)])
        assert np.abs(MK.reference_e2e(rec)["flows"] - np.load(os.path.join(GOLDEN, name + ".npz"))["flows"]).max() < 1e-5


def _one_gemm_volume(fmap1, fmap2p, f1, f2, a1, gamma):
    """float64 <A'[n], B'[m]> with A' and B' built entry by entry from clamped indices (NCHW features, a1 [B, N, 25])."""
    b, c, h, w = fmap1.shape
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    a_parts, b_parts = [fmap1.reshape(b, c, h * w) / 16], [fmap2p.reshape(b, c, h * w)]
    for l in range(25):
        yy = (ys + l // 5 - 2).clamp(0, h - 1).reshape(-1)
        xx = (xs + l % 5 - 2).clamp(0, w - 1).reshape(-1)
        a_parts.append(gamma * a1[:, None, :, l] * f1[:, :, yy, xx] / 16)
        b_parts.append(f2[:, :, yy, xx])
    A, Bm = torch.cat(a_parts, 1), torch.cat(b_parts, 1)  # [B, 6656, N]
    assert A.shape[1] == 6656
    return torch.bmm(A.transpose(1, 2), Bm).reshape(b * h * w, 1, h, w)


@pytest.mark.parametrize("h, w", [(3, 4), (5, 5), (7, 9)])
def test_volume_is_one_gemm_of_k_6656(h, w):
    """volume = <fmap1, fmap2'> / 16 + gamma corr2 equals A' B'^T in float64, on grids smaller than, equal to and larger than the
    5 x 5 window; against the reference's ShiftLSA + CorrBlock.corr where its checkout exists, else against the oracle."""
    g = torch.Generator().manual_seed(h * 10 + w)
    b = 2
    fmap1, fmap2p = (torch.randn(b, 256, h, w, generator=g, dtype=torch.float64) for _ in range(2))
    w1, w2 = (torch.randn(256, 256, 1, 1, generator=g, dtype=torch.float64) / 16 for _ in range(2))
    a1 = torch.softmax(torch.randn(b, h * w, 25, generator=g, dtype=torch.float64), -1)
    gamma = 0.7
    f1, f2 = torch.nn.functional.conv2d(fmap1, w1), torch.nn.functional.conv2d(fmap2p, w2)
    got = _one_gemm_volume(fmap1, fmap2p, f1, f2, a1, gamma)
    if ref_shim.available():
        import make_llaflow_golden as MK

        MK.load_llaflow()
        agg = sys.modules["ptlflow.models.llaflow.aggregate"]
        corr = sys.modules["ptlflow.models.llaflow.corr"]
        s = agg.ShiftLSA(dim=256, heads=1, size=5).double()
        s.to_f1.weight.data.copy_(w1)
        s.to_f2.weight.data.copy_(w2)
        with torch.no_grad():
            ref = corr.CorrBlock.corr(fmap1, fmap2p) + gamma * s(a1[:, None], fmap1, fmap2p)
    else:
        sd = {"s_lsa.to_f1.weight": w1, "s_lsa.to_f2.weight": w2}
        ref = LL.O.corr_volume(fmap1, fmap2p) + gamma * LL.shift_corr(a1, fmap1, fmap2p, sd)
    ref = ref.reshape(b * h * w, 1, h, w)
    assert (got - ref).abs().max().item() < 1e-12 * max(1.0, ref.abs().max().item())


def test_state_dict_contract_and_checkpoints():
    import ptlflow_b200 as pb

    for name, n in (("llaflow", 189), ("llaflow_raft", 186)):
        m = pb.get_model(name)
        sd = m.state_dict()
        assert {k: tuple(v.shape) for k, v in sd.items()} == LL.state_dict_shapes(name)
        assert len(sd) == n
        for k in ("ls1.to_qk.weight", "ls2.to_qk.weight", "s_lsa.to_f1.weight", "s_lsa.to_f2.weight", "lsa.to_v.weight", "lsa.gamma", "gamma"):
            assert k in sd, k
        assert ("att.to_qk.weight" in sd) == (name == "llaflow") and not any("pos_emb" in k for k in sd)
        m.load_state_dict(LL.synth_state_dict(name, 4, 1), strict=True)
        assert set(m.pretrained_checkpoints) == {"chairs", "things", "sintel", "kitti"}


def test_registry_defaults_and_gamma_clash():
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib as L, get_trainable_model_names
    from ptlflow_b200.models.llaflow.llaflow import llaflow, llaflow_raft

    for name, cls, gma in (("llaflow", llaflow, True), ("llaflow_raft", llaflow_raft, False)):
        assert name in pb.get_model_names() and name in get_trainable_model_names()
        m = cls()  # (the live-reference test's shim registers the reference's classes under the same names)
        assert (m.iters, m.corr_levels, m.corr_radius, m.dropout, m.max_flow, m.alternate_corr, m.gma) == (32, 4, 4, 0.0, 400, False, gma)
        assert m._variant == (L.VARIANT_GMA if gma else L.VARIANT_RAFT)
        # the keyword gamma is the loss decay (hparams); the attribute / state_dict key is the volume's parameter, initialised to 0
        assert m.hparams.gamma == 0.8 and m.loss_fn.gamma == 0.8
        assert isinstance(m.gamma, torch.nn.Parameter) and m.gamma.shape == (1,) and m.gamma.item() == 0.0
        assert m.lsa.gamma.item() == 0.0
        assert set(vars(m.hparams)) >= {"corr_levels", "corr_radius", "dropout", "gamma", "max_flow", "iters", "alternate_corr", "gma"}
    m = llaflow(corr_radius=3, iters=5, gma=False, alternate_corr=True, gamma=0.5)
    assert m.update_block.encoder.convc1.in_channels == 4 * 49 and m.att is None and m.hparams.gamma == 0.5 and m.alternate_corr


@pytest.mark.parametrize("kw, match", [(dict(corr_levels=3), "4 levels"), (dict(corr_levels=5), "4 levels"), (dict(iters=0), "iters")])
def test_constructor_refuses_what_the_reference_cannot_run(kw, match):
    from ptlflow_b200.models.llaflow.llaflow import llaflow, llaflow_raft

    for cls in (llaflow, llaflow_raft):
        with pytest.raises(ValueError, match=match):
            cls(**kw)


@pytest.mark.parametrize("h, w", [(96, 128), (128, 96), (120, 1024), (16, 16)])
def test_grid_limits_raise(h, w):
    """1/8 grids (after padding) under 2**corr_levels = 16 pixels per side, where the reference's bilinear_sampler divides by zero."""
    import ptlflow_b200 as pb

    m = pb.get_model("llaflow_raft").eval()
    with pytest.raises(ValueError, match="llaflow needs"):
        m._check_grid(-(-h // 8), -(-w // 8))
    m._check_grid(16, 16)
    m._check_grid(-(-121 // 8), 128)


def test_a22_argument_checks():
    L = _lib()
    lib = L.load()
    p = C.c_void_p(16)
    # (qk, a1, a2, B, H, W, dtype, stream)
    ok = [p, p, p, 1, 9, 11, 1, None]
    for i, bad in ((0, None), (2, None), (3, 0), (5, 0), (6, 3)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_local_similar(*args) == -1, (i, bad)
    # (fmap2, v, a2, gamma, out, B, H, W, dtype, stream)
    ok = [p, p, p, 0.5, p, 1, 9, 11, 1, None]
    for i, bad in ((1, None), (4, None), (6, -1), (8, 7)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_local_aggregate(*args) == -1, (i, bad)
    # (fmap1, f1, a1, fmap2, f2, gamma, a_pack, b_pad, b_pack, B, H, W, dtype, stream)
    ok = [p, p, p, p, p, 0.5, p, p, None, 1, 9, 11, 1, None]
    for i, bad in ((1, None), (4, None), (9, 0), (12, 4)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_shift_pack(*args) == -1, (i, bad)
    args = list(ok)
    args[6] = args[7] = None
    assert lib.pfb_shift_pack(*args) == -1  # nothing to write
    # (a_pack, b_pad, pyramid, B, H, W, levels, dtype, stream)
    pyr = (C.c_void_p * 4)(16, 16, 16, 16)
    ok = [p, p, pyr, 1, 16, 20, 4, 1, None]
    for i, bad in ((0, None), (1, C.c_void_p(8)), (6, 0), (6, 5), (4, 7), (7, 0)):
        args = list(ok)
        args[i] = bad
        assert lib.pfb_shift_volume_tiled(*args) == -1, (i, bad)
