"""GPU: MS-RAFT+ against the oracle and the reference vectors.

Kernels: group norm (+ ReLU, + residual, with the producer's bias) against F.group_norm in fp32 / f16 / bf16 for every width the
encoders use, also on inputs with a large common mean; the resize into the concat buffer against F.interpolate + torch.cat; both
convex 2x modes and downflow against the oracle, border pixels included; the 2-level on-the-fly lookup at C = 64, 96 (rows padded to
128), 128 and 256 on the tensor cores against the SIMT kernel and the oracle, with far-out-of-range coordinates.  Update block: one
iteration against the oracle on the tensor path and with kernel_impl = 1.  End to end: the e2e_ms_raft_p_* vectors in fp32 (eager
and graph replay), the default model at 436x1024 in f16 / bf16 against the fp32 model, graph replay against eager, and the volume
path against the on-the-fly one.
"""
import json
import math
import os
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import ms_raft_oracle as MS
from helpers import load_golden
from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = os.environ.get("PFB_PARITY_REPORT")  # optional: one JSON line of measured errors per check
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
EPS = {torch.float32: 1e-6, torch.float16: 1e-3, torch.bfloat16: 8e-3}  # storage rounding unit


def _report(**kw):
    if not REPORT:
        return
    try:
        os.makedirs(os.path.dirname(REPORT), exist_ok=True)
        with open(REPORT, "a") as f:
            f.write(json.dumps(kw) + "\n")
    except OSError:
        pass


def _gen(name, shape, seed=0, scale=1.0):
    return torch.from_numpy(synth.synth_normal(name, shape, seed, scale=scale))


def _model(kwargs, sd, dtype=torch.float32, impl=0):
    import ptlflow_b200 as pb

    model = pb.get_model("ms_raft_p", args=Namespace(model=Namespace(**kwargs)))
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    model = model.eval().to(DEV)
    if dtype != torch.float32:
        model = model.to(dtype)
    model.kernel_impl = impl
    return model


def _pm(t):
    return t.permute(0, 2, 3, 1).contiguous()


# --------------------------------------------------------------------------------------
# group norm, resize into the concat buffer, convex 2x, downflow
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C", [64, 96, 128, 160, 256])
@pytest.mark.parametrize("mode", ["relu", "residual", "plain"])
def test_group_norm_vs_torch(C, dtype, mode):
    from ptlflow_b200 import ops

    x = _gen(f"gn/x{C}", (2, C, 13, 21), scale=2.0) + 0.5
    bias, g, b = _gen(f"gn/b{C}", (C,), scale=0.7), 1 + _gen(f"gn/g{C}", (C,), scale=0.2), _gen(f"gn/be{C}", (C,), scale=0.3)
    res = _gen(f"gn/r{C}", (2, C, 13, 21))
    xq, rq = x.to(dtype).float(), res.to(dtype).float()
    ref = F.group_norm(xq + bias[None, :, None, None], C // 8, g, b, eps=1e-5)
    if mode != "plain":
        ref = torch.relu(ref)
    if mode == "residual":
        ref = torch.relu(rq + ref)
    out = ops.group_norm_act(_pm(xq).to(DEV, dtype), g.to(DEV), b.to(DEV), 8, bias=bias.to(DEV), relu=mode != "plain",
                             residual=_pm(rq).to(DEV, dtype) if mode == "residual" else None)
    d = (out.float().cpu().permute(0, 3, 1, 2) - ref).abs().max().item()
    _report(test="ms_group_norm", C=C, dtype=str(dtype), mode=mode, err=d)
    assert d < 4 * EPS[dtype] * max(1.0, ref.abs().max().item()), d


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=lambda d: str(d)[6:])
def test_group_norm_large_common_mean_and_first_conv_sums(dtype):
    """A common mean 50x the spread (sums accumulated per channel in fp32, combined per group in fp64), and the group norm applied
    from sums a producer accumulated (the first convolution's epilogue)."""
    from ptlflow_b200 import ops

    x = 50.0 + _gen("gn/mean", (2, 64, 48, 64))
    g, b = 1 + _gen("gn/mg", (64,), scale=0.2), _gen("gn/mb", (64,), scale=0.3)
    xq = x.to(dtype).float()
    ref = F.group_norm(xq, 8, g, b, eps=1e-5)
    xd = _pm(xq).to(DEV, dtype)
    out = ops.group_norm_act(xd, g.to(DEV), b.to(DEV), 8, relu=False)
    ws = ops.instance_norm_workspace(xd.shape, xd.device)
    s = xd.float().sum(dim=(1, 2)).double()
    q = (xd.float().double() ** 2).sum(dim=(1, 2))
    ws[: 2 * 64 * 2].copy_(torch.stack([s, q], -1).reshape(-1))
    out2 = ops.group_norm_act(xd, g.to(DEV), b.to(DEV), 8, relu=False, stats_ws=ws)
    d = (out.float().cpu().permute(0, 3, 1, 2) - ref).abs().max().item()
    d2 = (out2.float().cpu().permute(0, 3, 1, 2) - ref).abs().max().item()
    _report(test="ms_group_norm_mean", dtype=str(dtype), err=d, err_apply=d2)
    tol = 2e-3 if dtype == torch.float32 else 4e-2
    assert d < tol and d2 < tol, (d, d2)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("cs,ck,h,w", [(256, 128, 4, 6), (128, 96, 7, 9), (96, 64, 1, 3), (256, 64, 13, 32)])
def test_upsample2x_concat_vs_interpolate(cs, ck, h, w, dtype):
    from ptlflow_b200 import ops

    src = _gen(f"up/s{cs}", (2, cs, h, w)).to(dtype)
    skip = _gen(f"up/k{ck}", (2, ck, 2 * h, 2 * w)).to(dtype)
    ref = torch.cat([F.interpolate(src.float(), scale_factor=2, mode="bilinear", align_corners=False), skip.float()], 1)
    out = ops.upsample2x_concat(_pm(src).to(DEV), _pm(skip).to(DEV))
    d = (out.float().cpu().permute(0, 3, 1, 2) - ref).abs().max().item()
    assert d <= EPS[dtype] * 4, d


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_convex_upsample2x_both_modes_and_downflow(dtype):
    from ptlflow_b200 import ops

    b, h, w = 2, 7, 11
    coords = O.coords_grid(b, h, w) + _gen("cx/c", (b, 2, h, w), scale=30.0)
    mask = _gen("cx/m", (b, 36, h, w), scale=2.0).to(dtype).float()
    cd, md = _pm(coords).to(DEV), _pm(mask).to(DEV, dtype)
    ref_flow = MS.convex_up2(coords - O.coords_grid(b, h, w), mask)
    ref_coords = MS.convex_up2(coords, mask)
    flow = ops.convex_upsample2x(cd, md, 0, (2 * h - 3, 2 * w - 1), (1, 1)).cpu()
    nxt = ops.convex_upsample2x(cd, md, 1).cpu().permute(0, 3, 1, 2)
    e_flow = (flow - ref_flow[:, :, 1 : 2 * h - 2, 1 : 2 * w]).abs().max().item()
    e_coords = (nxt - ref_coords).abs().max().item()
    border = (nxt - ref_coords)[..., [0, -1], :].abs().max().item()
    small = ops.downflow(ref_flow.contiguous().to(DEV), (h // 2, w // 3)).cpu()
    ref_small = F.interpolate(ref_flow, size=(h // 2, w // 3), mode="bilinear", align_corners=True)
    ref_small = torch.cat([ref_small[:, :1] * ((w // 3) / (2 * w)), ref_small[:, 1:] * ((h // 2) / (2 * h))], 1)
    e_small = (small - ref_small).abs().max().item()
    _report(test="ms_convex2x", dtype=str(dtype), err_flow=e_flow, err_coords=e_coords, err_small=e_small)
    scale = ref_coords.abs().max().item()
    assert e_flow < 1e-5 * scale and e_coords < 1e-5 * scale and border < 1e-5 * scale and e_small < 1e-5 * scale


# --------------------------------------------------------------------------------------
# 2-level on-the-fly lookup at every feature width
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C", [64, 96, 128, 256])
def test_onthefly_lookup_two_levels(C, dtype):
    from ptlflow_b200 import ops

    b, h, w = 2, 24, 40
    f1 = _gen(f"otf/f1_{C}", (b, C, h, w)).to(dtype).float()
    f2 = _gen(f"otf/f2_{C}", (b, C, h, w)).to(dtype).float()
    coords = O.coords_grid(b, h, w) + _gen(f"otf/c{C}", (b, 2, h, w), scale=3.0)
    coords[0, :, :3] += 400.0  # far out of range: flagged queries for the SIMT pass
    coords[1, 0, 5:9, 5:9] -= 1e4
    ref = O.alt_corr_lookup(f1, f2, coords, 4, 2)
    cd = _pm(coords).to(DEV)
    a, bb = _pm(f1).to(DEV, dtype), _pm(f2).to(DEV, dtype)
    simt = ops.corr_lookup_onthefly_scaled(a, ops.feature_pyramid(bb, 2), cd, 4, 1 / math.sqrt(C), False)
    if C % 64:
        a, bb = F.pad(a, (0, 64 - C % 64)).contiguous(), F.pad(bb, (0, 64 - C % 64)).contiguous()
    tc = ops.corr_lookup_onthefly_scaled(a, ops.feature_pyramid(bb, 2), cd, 4, 1 / math.sqrt(C), True)
    flagged = int(tc._pfb_flags.sum().item())
    r = ref.permute(0, 2, 3, 1)
    e_tc = (tc[..., :162].float().cpu() - r).abs().max().item()
    e_simt = (simt[..., :162].float().cpu() - r).abs().max().item()
    _report(test="ms_onthefly", C=C, dtype=str(dtype), err_tc=e_tc, err_simt=e_simt, flagged=flagged)
    tol = 4 * EPS[dtype] * max(1.0, r.abs().max().item())
    assert flagged > 0 and e_tc < tol and e_simt < tol, (e_tc, e_simt, flagged)
    assert (tc[..., 162:] == 0).all()


# --------------------------------------------------------------------------------------
# one update iteration
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,impl", [(torch.float32, 0), (torch.float16, 0), (torch.bfloat16, 0), (torch.float16, 1)])
def test_update_iteration_vs_oracle(dtype, impl):
    import ptlflow_b200 as pb
    from ptlflow_b200 import ops
    from ptlflow_b200.engine import MSRaftEngine

    sd, x = MS.op_inputs()
    q = lambda t: t.to(dtype).float()  # noqa: E731
    net, inp, corr, flow = q(x["net"]), q(x["inp"]), q(x["corr"]), q(x["flow"])
    with O.fp32_strict():
        n_ref, m_ref, d_ref = MS.update_block(net, inp, corr, flow, sd)
    model = pb.get_model("ms_raft_p")
    model.load_state_dict(sd)
    model = model.to(DEV, dtype)
    eng = MSRaftEngine(model.update_block, 5, 128, 128, 2, 4, dtype, torch.device(DEV), impl=impl)
    b, _, h, w = net.shape
    coords0 = O.coords_grid(b, h, w)
    coords = ops.coords_to_pixel_major(coords0 + flow).to(DEV)
    net_d = _pm(net).to(DEV, dtype)
    with torch.no_grad():
        mask = eng.update_iter(net_d, _pm(inp).to(DEV, dtype), coords, corr=_pm(corr).to(DEV, dtype), want_mask=True)
    torch.cuda.synchronize()
    e_net = (net_d.float().cpu().permute(0, 3, 1, 2) - n_ref).abs().max().item()
    e_delta = ((coords.cpu().permute(0, 3, 1, 2) - coords0 - flow) - d_ref).abs().max().item()
    e_mask = (mask.float().cpu().permute(0, 3, 1, 2) - m_ref).abs().max().item()
    _report(test="ms_update_iter", dtype=str(dtype), impl=impl, err_net=e_net, err_delta=e_delta, err_mask=e_mask)
    # about 4x what one H100 80GB HBM3 (400 W) measured: fp32 <= 8e-7; f16 1.0e-3 / 1.3e-4 / 4.4e-5 and bf16 7.4e-3 / 1.1e-3 / 3.7e-4
    # on net / delta / mask
    tol = {torch.float32: (1e-5, 1e-5, 1e-5), torch.float16: (4e-3, 5e-4, 2e-4), torch.bfloat16: (3e-2, 4e-3, 1.5e-3)}[dtype]
    assert e_net < tol[0] and e_delta < tol[1] and e_mask < tol[2], (e_net, e_delta, e_mask)


# --------------------------------------------------------------------------------------
# end to end
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", MS.E2E)
def test_fp32_matches_reference_vectors(name):
    recipe, g = load_golden(name)
    sd, img, kw = MS.e2e_inputs(recipe)
    model = _model(kw, sd)
    inputs = {"images": img.to(DEV)}
    if recipe["warm"]:
        inputs["prev_preds"] = {"flow_small": torch.from_numpy(g["prev_flow_small"]).to(DEV)}
    with torch.no_grad():
        out = model(inputs)
        out2 = model(inputs)  # captures, then replays the CUDA graph
        out3 = model(inputs)
    assert model.graph_replays >= 1
    err = np.abs(out["flows"].cpu().numpy() - g["flows"]).max()
    err_replay = max(np.abs(o["flows"].cpu().numpy() - g["flows"]).max() for o in (out2, out3))
    err_small = np.abs(out["flow_small"].cpu().numpy() - g["flow_small"]).max()
    _report(test="ms_fp32_golden", case=name, err_flow=float(err), err_replay=float(err_replay), err_flow_small=float(err_small),
            max_flow=float(np.abs(g["flows"]).max()))
    assert out["flows"].shape == g["flows"].shape and out["flow_small"].shape == g["flow_small"].shape
    assert err < 1e-3 and err_replay < 1e-3 and err_small < 1e-3, f"{name}: max-abs flow error {err} / replay {err_replay} / small {err_small}"


def test_half_model_one_graph_per_forward_and_training_guard():
    recipe, g = load_golden("e2e_ms_raft_p_ragged_b2")
    sd, img, kw = MS.e2e_inputs(recipe)
    model = _model(kw, sd, torch.float16)
    with torch.no_grad():
        for _ in range(3):
            out = model({"images": img.to(DEV).half()})
    assert model.graph_replays >= 1 and len(model._graphs) == 1
    assert out["flows"].shape == g["flows"].shape and out["flows"].dtype == torch.float16
    assert out["flow_small"].shape == g["flow_small"].shape
    d = np.abs(out["flows_fp32"].cpu().numpy() - g["flows"])
    _report(test="ms_f16_vs_fp32_ref", err_flow=float(d.max()), mean_err=float(d.mean()), max_flow=float(np.abs(g["flows"]).max()))
    assert d.max() < 0.05 and d.mean() < 0.01, (d.max(), d.mean())  # measured 0.014 / 0.0034 (|flow| <= 120)
    model.train()
    with pytest.raises(NotImplementedError):
        model({"images": img.to(DEV).half()})


# Half precision at 436x1024 against the fp32 model on the same GPU (TF32 off; the fp32 model matches the reference vectors to
# < 5e-5 px above).  The fp32 oracle itself cannot run at this size: its all-pairs lookup at 1/2 scale is a 114688^2 volume.
# Gates about 3x above what one H100 80GB HBM3 (400 W) measured, as fractions of max |flow| (789 px with these random weights):
#   f16 max-abs 0.018 px (2.3e-5), mean-abs 0.0036 px (4.5e-6);  bf16 max-abs 0.153 px (1.9e-4), mean-abs 0.031 px (3.9e-5)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=lambda d: str(d)[6:])
def test_sintel_size_against_fp32(dtype):
    sd = MS.synth_state_dict(MS.state_dict_shapes(), 1234)
    img = torch.from_numpy(synth.synth_images(1, 436, 1024, 4321, "smooth")).to(DEV)
    ref_model = _model({}, sd)
    with torch.no_grad(), O.fp32_strict():
        ref = ref_model({"images": img})["flows_fp32"].float().cpu()
    del ref_model
    torch.cuda.empty_cache()
    model = _model({}, sd, dtype)
    with torch.no_grad():
        out = model({"images": img.to(dtype)})
    d = (out["flows_fp32"].float().cpu() - ref).abs()
    mag = ref.abs().max().item()
    _report(test="ms_sintel_size", dtype=str(dtype), err_flow=d.max().item(), mean_err=d.mean().item(), max_flow=mag)
    gate_max, gate_mean = {torch.float16: (8e-5, 1.5e-5), torch.bfloat16: (6e-4, 1.2e-4)}[dtype]
    assert d.max().item() < gate_max * mag and d.mean().item() < gate_mean * mag, \
        f"max-abs {d.max().item():.4g} mean-abs {d.mean().item():.4g} (|flow| <= {mag:.1f})"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=lambda d: str(d)[6:])
def test_graph_replay_matches_eager(dtype):
    recipe, _ = load_golden("e2e_ms_raft_p_ragged_b2")
    sd, img, kw = MS.e2e_inputs(recipe)
    model = _model(kw, sd, dtype)
    x = img.to(DEV, dtype)
    with torch.no_grad():
        model.use_cuda_graph = False
        eager = model({"images": x})["flows_fp32"].clone()
        model.use_cuda_graph = True
        model({"images": x})
        model({"images": x})
        replay = model({"images": x})["flows_fp32"]
    assert model.graph_replays >= 2
    d = (eager - replay).abs().max().item()
    _report(test="ms_graph_vs_eager", dtype=str(dtype), err=d)
    assert d < (1e-4 if dtype == torch.float32 else 6e-2), d  # measured 3.1e-5 / 0.018


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=lambda d: str(d)[6:])
def test_volume_path_agrees_with_onthefly(dtype):
    recipe, _ = load_golden("e2e_ms_raft_p_default")
    sd, img, _ = MS.e2e_inputs(recipe)
    x = img.to(DEV, dtype)
    with torch.no_grad():
        a = _model({}, sd, dtype)({"images": x})["flows_fp32"]
        b = _model({"alternate_corr": False}, sd, dtype)({"images": x})["flows_fp32"]
    d = (a - b).abs()
    _report(test="ms_volume_vs_onthefly", dtype=str(dtype), err=d.max().item(), mean_err=d.mean().item())
    # measured: fp32 1.9e-5 / 2.4e-6, bf16 0.012 / 0.0024 (max / mean)
    assert d.max().item() < (1e-3 if dtype == torch.float32 else 0.05) and d.mean().item() < (1e-4 if dtype == torch.float32 else 0.01)


def test_host_errors_raise_before_any_launch():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    sd = MS.synth_state_dict(MS.state_dict_shapes(), 3)
    model = _model({}, sd)
    torch.cuda.synchronize()
    before = lib.pfb_launch_count(-1)
    with torch.no_grad():
        with pytest.raises(ValueError, match="multiples of 16"):
            model({"images": torch.rand(1, 2, 3, 100, 150, device=DEV), "prev_preds": {"flow_small": torch.zeros(1, 2, 6, 9, device=DEV)}})
        model.iters = (4, 6, 0, 10)
        with pytest.raises(ValueError, match="iters"):
            model({"images": torch.rand(1, 2, 3, 64, 96, device=DEV)})
        model.iters = (4, 6, 5, 10)
        with pytest.raises(ValueError, match="lookup_pyramid_levels"):
            model({"images": torch.rand(1, 2, 3, 16, 96, device=DEV)})
    assert lib.pfb_launch_count(-1) == before
