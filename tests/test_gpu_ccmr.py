"""GPU: CCMR / CCMR+'s new kernels against torch / the oracle, the update iteration in every dtype and impl, the fp32 fixtures
(eager and graph replay), half precision at 436x1024 against the fp32 model, the volume path and the host errors."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import ccmr_oracle as CC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(HERE, "golden")
TOL = {torch.float32: 1e-4, torch.float16: 2e-2, torch.bfloat16: 1e-1}


def _model(name, sd, dtype=torch.float32, **kw):
    import ptlflow_b200 as pb
    from argparse import Namespace

    m = pb.get_model(name, args=Namespace(model=Namespace(**kw)) if kw else None)
    m.load_state_dict(sd)
    return m.eval().to(DEV).to(dtype)


def _pm(x):  # NCHW -> pixel-major
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_layernorm_and_lpi_convolutions(dtype):
    from ptlflow_b200 import ops

    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 9, 13, 128, generator=g)
    gm, bt = 1 + 0.1 * torch.randn(128, generator=g), 0.1 * torch.randn(128, generator=g)
    xd = x.to(DEV, dtype)
    ref = F.layer_norm(xd.float().cpu(), (128,), gm, bt, eps=1e-6)
    assert (ops.layernorm(xd, gm.to(DEV), bt.to(DEV)).float().cpu() - ref).abs().max() < 4 * TOL[dtype]
    ref0 = F.layer_norm(xd.float().cpu(), (128,), eps=1e-6)
    assert (ops.layernorm(xd).float().cpu() - ref0).abs().max() < 4 * TOL[dtype]
    w, b = 0.3 * torch.randn(128, 1, 3, 3, generator=g), 0.1 * torch.randn(128, generator=g)
    wt = w.reshape(128, 9).t().contiguous().to(DEV)
    conv = F.conv2d(xd.float().cpu().permute(0, 3, 1, 2), w, b, padding=1, groups=128).permute(0, 2, 3, 1)
    out0 = ops.depthwise_conv3x3_ex(xd, wt, b.to(DEV), 0)
    assert (out0.float().cpu() - F.gelu(conv)).abs().max() < 4 * TOL[dtype]
    add = torch.randn(2, 9, 13, 128, generator=g).to(DEV, dtype)
    out1 = ops.depthwise_conv3x3_ex(xd, wt, b.to(DEV), 1, addend=add)
    assert (out1.float().cpu() - (conv + add.float().cpu())).abs().max() < 4 * TOL[dtype]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fourier_features(dtype):
    from ptlflow_b200 import ops

    sd = {"p.pos_embeder.token_projection.weight": torch.eye(64, 64)[:, :, None, None].repeat(2, 1, 1, 1)[:128],
          "p.pos_embeder.token_projection.bias": torch.zeros(128)}
    ref = CC.fourier_pos(sd, "p.", 1, 28, 64)[0, :, :64].reshape(28, 64, 64)
    out = ops.fourier_features(28, 64, dtype, DEV).float().cpu()
    assert (out - ref).abs().max() < (2e-6 if dtype == torch.float32 else 8e-3)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_xca_statistics_and_fold(dtype):
    from ptlflow_b200 import ops

    g = torch.Generator().manual_seed(1)
    B, N = 2, 114688  # ccmr_p's 1/2 scale of a 436x1024 pair padded to 448x1024
    qk = (torch.randn(B, N, 256, generator=g) + 0.3).to(DEV, dtype)
    st = ops.xca_stats(qk.view(B, 448 // 2, 1024 // 2, 256))
    q64 = qk.double()
    gram = torch.einsum("bnhi,bnhj->bhij", q64[..., :128].reshape(B, N, 8, 16), q64[..., 128:].reshape(B, N, 8, 16)).reshape(B, 2048)
    ref = torch.cat([gram, (q64[..., :128] ** 2).sum(1), (q64[..., 128:] ** 2).sum(1)], 1)
    rel = ((st.double() - ref).abs() / ref.abs().clamp_min(1.0)).max().item()
    assert rel < 1e-5, rel
    assert torch.equal(st, ops.xca_stats(qk.view(B, 224, 512, 256)))  # deterministic
    # fold against the explicit XCA on a small map
    Ns = 60
    q, k, v = (torch.randn(B, Ns, 128, generator=g) for _ in range(3))
    t = 1 + 0.3 * torch.randn(8, generator=g)
    wv, bv, wp, bp = torch.randn(128, 128, generator=g) / 11, 0.1 * torch.randn(128, generator=g), torch.randn(128, 128, generator=g) / 11, \
        0.1 * torch.randn(128, generator=g)
    stats = ops.xca_stats(torch.cat([q, k], -1).view(B, 6, 10, 256).to(DEV))
    w, wk, bias = ops.xca_fold(stats, t.to(DEV), wv.to(DEV), bv.to(DEV), wp.to(DEV), bp.to(DEV), dtype)
    ref = F.linear(CC.xca(q, k, F.linear(v, wv, bv), t), wp, bp)
    got = torch.einsum("bni,bio->bno", v.to(DEV, dtype).float(), w.float()).cpu() + bias.cpu()[:, None]
    assert (got - ref).abs().max() < 20 * TOL[dtype]
    if wk is not None:
        assert torch.equal(wk.view(B, 128, 128).transpose(1, 2).cpu(), w.cpu())


def test_handover_and_upflow2():
    from ptlflow_b200 import ops

    g = np.load(os.path.join(GOLDEN, "op_ccmr.npz"))
    _, x = CC.op_inputs()
    hand = ops.convex_handover2x(_pm(x["coords"]).to(DEV), _pm(x["mask"]).to(DEV))
    assert (hand.permute(0, 3, 1, 2).cpu() - torch.from_numpy(g["handover"])).abs().max() < 1e-4
    up = ops.upflow2(x["flow_lo"].to(DEV))
    assert (up.cpu() - torch.from_numpy(g["upflow2"])).abs().max() < 1e-4
    win = ops.upflow2(x["flow_lo"].to(DEV), out_hw=(7, 11), pad=(2, 1))
    assert torch.equal(win, up[:, :, 2:9, 1:12])


def _engine(dtype, impl=0):
    from ptlflow_b200.engine import CCMREngine

    sd, x = CC.op_inputs()
    m = _model("ccmr_p", sd, dtype)
    m.kernel_impl = impl
    return m, m._get_engine(dtype, torch.device(DEV)), sd, x


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_xcit_context_matches_reference(dtype):
    m, eng, sd, x = _engine(dtype)
    g = np.load(os.path.join(GOLDEN, "op_ccmr.npz"))
    out = eng.xcit_context(1, _pm(x["ctx"]).to(DEV, dtype)).permute(0, 3, 1, 2).float().cpu()
    err = (out - torch.from_numpy(g["xcit_self"])).abs().max().item()
    assert err < {torch.float32: 1e-3, torch.float16: 3e-2, torch.bfloat16: 2e-1}[dtype], err


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_update_iteration_matches_oracle(dtype, impl):
    if dtype == torch.float32 and impl == 0:
        pytest.skip("fp32 runs on SIMT under every impl")
    m, eng, sd, x = _engine(dtype, impl)
    with torch.no_grad():
        gc = CC.xcit(sd, "xcit.1.", x["inp"])
        net_r, mask_r, delta_r = CC.update_block(x["net"], x["inp"], x["corr"], x["flow"], gc, sd, 1)
    net = _pm(x["net"]).to(DEV, dtype)
    coords = _pm(CC.O.coords_grid(2, 6, 9) + x["flow"]).to(DEV)
    corr = _pm(x["corr"]).to(DEV, dtype)
    mask = eng.update_iter(net, _pm(x["inp"]).to(DEV, dtype), coords, corr=corr, want_mask=True, scale=1)
    tol = {torch.float32: 1e-3, torch.float16: 5e-2, torch.bfloat16: 3e-1}[dtype]
    assert (net.permute(0, 3, 1, 2).float().cpu() - net_r).abs().max() < tol
    assert (mask.permute(0, 3, 1, 2).float().cpu() - mask_r).abs().max() < 4 * tol
    delta = coords.permute(0, 3, 1, 2).cpu() - CC.O.coords_grid(2, 6, 9) - x["flow"]
    assert (delta - delta_r).abs().max() < 4 * tol


@pytest.mark.parametrize("name", CC.E2E)
def test_fp32_fixtures_eager_and_replayed(name):
    rec = CC.recipe_of(CC.E2E_CASES[CC.E2E.index(name)])
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    sd, img, kw = CC.e2e_inputs(rec)
    m = _model(rec["model"], sd, **kw)
    inputs = {"images": img.to(DEV)}
    if rec["warm"]:
        inputs["prev_preds"] = {"flow_small": torch.from_numpy(g["prev_flow_small"]).to(DEV)}
    outs = []
    with torch.no_grad():
        for _ in range(3):  # eager, eager + capture, replay
            outs.append(m(inputs))
    assert m.graph_replays >= 1
    for o in outs:
        assert (o["flows"].cpu() - torch.from_numpy(g["flows"])).abs().max().item() < 1e-3
        assert (o["flow_small"].cpu() - torch.from_numpy(g["flow_small"])).abs().max().item() < 1e-3
    # graph replay against the first, eager forward (cuDNN's encoder convolutions are not bitwise deterministic)
    assert (outs[0]["flows"] - outs[2]["flows"]).abs().max().item() < 1e-4


def test_half_precision_at_full_size():
    sd = CC.synth_state_dict(CC.state_dict_shapes("ccmr_p"), 5)
    img = torch.from_numpy(CC.synth.synth_images(1, 436, 1024, 6, "smooth")).to(DEV)
    with torch.no_grad():
        ref = _model("ccmr_p", sd)({"images": img})["flows"].float()
        # measured on an H100 80GB HBM3 (700 W): f16 0.044 / 0.0093 px, bf16 0.39 / 0.069 px max-abs / mean-abs, max |flow| 70.6 px
        for dtype, bound in ((torch.float16, (0.15, 0.03)), (torch.bfloat16, (1.2, 0.2))):
            out = _model("ccmr_p", sd, dtype)({"images": img.to(dtype)})["flows_fp32"].float()
            e = (out - ref).abs()
            print(f"ccmr_p {dtype} at 436x1024: max-abs {e.max().item():.4f} mean-abs {e.mean().item():.5f} px "
                  f"(max |flow| {ref.abs().max().item():.1f})")
            assert e.max().item() < bound[0] and e.mean().item() < bound[1]


def test_volume_path_agrees_with_on_the_fly():
    sd = CC.synth_state_dict(CC.state_dict_shapes("ccmr"), 8)
    img = torch.from_numpy(CC.synth.synth_images(1, 96, 128, 9, "smooth")).to(DEV)
    with torch.no_grad():
        a = _model("ccmr", sd, iters=(2, 2, 2))({"images": img})["flows"]
        b = _model("ccmr", sd, iters=(2, 2, 2), alternate_corr=False)({"images": img})["flows"]
    assert (a - b).abs().max().item() < 1e-3


def test_host_errors_before_any_launch():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    sd = CC.synth_state_dict(CC.state_dict_shapes("ccmr"), 1)
    m = _model("ccmr", sd)
    n0 = lib.pfb_launch_count(-1)
    with pytest.raises(ValueError, match="multiples of 32"):
        m({"images": torch.zeros(1, 2, 3, 80, 96, device=DEV), "prev_preds": {"flow_small": torch.zeros(1, 2, 5, 6, device=DEV)}})
    m.iters = (1, 2)
    with pytest.raises(ValueError, match="iters"):
        m({"images": torch.zeros(1, 2, 3, 64, 96, device=DEV)})
    m.iters = (1, 1, 1)
    m.train()
    with pytest.raises(NotImplementedError):
        with torch.enable_grad():
            m({"images": torch.zeros(1, 2, 3, 64, 96, device=DEV)})
    assert lib.pfb_launch_count(-1) == n0
