"""GPU parity tests, operator level: every call goes through the C ABI (ptlflow_b200.ops -> ctypes).

The oracle (oracle/raft_oracle.py, pinned to the reference by tests/test_oracle_golden.py) and the
committed reference vectors (tests/golden) are the checkers.  Tolerances: fp32 storage <= 1e-4 on
operators (bit-level agreement is not defined across different fp32 summation orders); f16/bf16
storage is compared to the fp32 oracle with the tolerance written in each test.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden
from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _ops():
    from ptlflow_b200 import ops

    return ops


def _nhwc(x, dtype=torch.float32):
    return x.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)


def _golden_fmaps(recipe):
    b, c, h, w = recipe["b"], recipe["c"], recipe["h"], recipe["w"]
    f1 = torch.from_numpy(synth.synth_normal("ops/fmap1", (b, c, h, w), recipe["seed"]))
    f2 = torch.from_numpy(synth.synth_normal("ops/fmap2", (b, c, h, w), recipe["seed"]))
    return f1, f2


# ------------------------------------------------------------------------------------------
# a1 + a2 + a3
# ------------------------------------------------------------------------------------------
def test_library_loads_on_device():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    assert lib.pfb_version() >= 100
    assert lib.pfb_device_arch() == 90, "expected an sm_90 (Hopper) device"


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.float16, 2e-2), (torch.bfloat16, 1.5e-1)])
def test_volume_pyramid_lookup_vs_reference_vectors(dtype, tol):
    ops = _ops()
    recipe, g = load_golden("op_corr_lookup")
    f1, f2 = _golden_fmaps(recipe)
    pyr = ops.corr_volume_build(_nhwc(f1, dtype), _nhwc(f2, dtype), recipe["levels"], impl=1)
    assert [list(p.shape[-2:]) for p in pyr] == g["level_shapes"].tolist()
    ref_pyr = O.corr_pyramid(O.corr_volume(f1, f2), recipe["levels"])
    for p, r in zip(pyr, ref_pyr):
        assert (p.float().cpu() - r[:, 0]).abs().max().item() < tol
    assert np.abs(pyr[3].float().cpu().numpy()[:, None] - g["level3"]).max() < tol
    coords = torch.from_numpy(g["coords"])
    look = ops.corr_lookup(pyr, _nhwc(coords), recipe["radius"], (recipe["h"], recipe["w"]), nchw=True, out_dtype=torch.float32)
    assert look.shape == g["lookup"].shape
    assert np.abs(look.cpu().numpy() - g["lookup"]).max() < tol * 2
    # pixel-major layout with zero-filled pad columns returns the same numbers
    planes = g["lookup"].shape[1]
    look2 = ops.corr_lookup(pyr, _nhwc(coords), recipe["radius"], (recipe["h"], recipe["w"]), nchw=False, out_dtype=torch.float32, out_stride=planes + 60)
    assert (look2[..., :planes].permute(0, 3, 1, 2) - look).abs().max().item() < 1e-5  # fast path (r<=4) vs generic kernel
    assert look2[..., planes:].abs().max().item() == 0.0


@pytest.mark.parametrize("radius,levels", [(4, 4), (3, 4), (1, 1), (0, 2), (5, 3)])
def test_lookup_radius_and_levels(radius, levels):
    ops = _ops()
    b, c, h, w = 1, 32, 16, 24
    f1 = torch.from_numpy(synth.synth_normal("rl/f1", (b, c, h, w), 5))
    f2 = torch.from_numpy(synth.synth_normal("rl/f2", (b, c, h, w), 5))
    coords = O.coords_grid(b, h, w) + torch.from_numpy(synth.synth_normal("rl/c", (b, 2, h, w), 5, scale=5.0))
    pyr = ops.corr_volume_build(_nhwc(f1), _nhwc(f2), levels, impl=1)
    look = ops.corr_lookup(pyr, _nhwc(coords), radius, (h, w))
    ref = O.corr_lookup(O.corr_pyramid(O.corr_volume(f1, f2), levels), coords, radius)
    assert (look.cpu() - ref).abs().max().item() < 3e-5


def test_lookup_rejects_bad_arguments():
    ops = _ops()
    f = torch.zeros(1, 8, 8, 16, device=DEV)
    with pytest.raises(RuntimeError):
        ops.corr_volume_build(f, f, levels=5)  # 8x8 grid cannot hold 5 levels
    with pytest.raises(RuntimeError):
        ops.corr_volume_build(f.cpu(), f.cpu(), levels=1)  # CPU tensor: loud failure, no fallback
    pyr = ops.corr_volume_build(f, f, 2)
    with pytest.raises(RuntimeError):
        ops.corr_lookup(pyr, torch.zeros(1, 8, 8, 2, device=DEV, dtype=torch.float16), 4, (8, 8))


# ------------------------------------------------------------------------------------------
# a4: on-the-fly and the plugin entry point
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-5), (torch.float16, 3e-2)])
def test_onthefly_vs_reference_vectors(dtype, tol):
    ops = _ops()
    recipe, g = load_golden("op_alt_corr")
    f1, f2 = _golden_fmaps(recipe)
    fpyr = ops.feature_pyramid(_nhwc(f2, dtype), recipe["levels"])
    look = ops.corr_lookup_onthefly(_nhwc(f1, dtype), fpyr, _nhwc(torch.from_numpy(g["coords"])), recipe["radius"], out_dtype=torch.float32)
    assert np.abs(look.cpu().numpy() - g["lookup"]).max() < tol


def test_alt_cuda_corr_plugin_contract():
    """Same call as the reference's pybind module (correlation.cpp:23-33)."""
    from ptlflow_b200 import alt_cuda_corr

    b, c, h1, w1, h2, w2, r = 2, 32, 9, 14, 5, 7, 3
    f1 = torch.from_numpy(synth.synth_normal("p/f1", (b, h1, w1, c), 9))
    f2 = torch.from_numpy(synth.synth_normal("p/f2", (b, h2, w2, c), 9))
    coords = torch.from_numpy(synth.synth_normal("p/c", (b, 1, h1, w1, 2), 9, scale=4.0)) + 2.0
    (out,) = alt_cuda_corr.forward(f1.to(DEV), f2.to(DEV), coords.to(DEV), r)
    ref = O.alt_cuda_corr_forward(f1, f2, coords, r)
    assert out.shape == ref.shape == (b, 1, (2 * r + 1) ** 2, h1, w1)
    assert (out.cpu() - ref).abs().max().item() < 5e-5
    with pytest.raises(RuntimeError):  # CHECK_INPUT semantics
        alt_cuda_corr.forward(f1, f2.to(DEV), coords.to(DEV), r)
    with pytest.raises(RuntimeError):
        alt_cuda_corr.forward(f1.to(DEV).permute(0, 2, 1, 3), f2.to(DEV), coords.to(DEV), r)


# ------------------------------------------------------------------------------------------
# conv building block
# ------------------------------------------------------------------------------------------
CONV_CASES = [
    # (srcs channels, Cout, KH, KW, epilogue)
    ([324], 256, 1, 1, "relu"),
    ([256], 192, 3, 3, "relu"),
    ([2], 128, 7, 7, "relu"),
    ([128, 128, 128], 256, 1, 5, "linear"),
    ([96, 64, 82], 96, 3, 3, "linear"),
    ([128], 2, 3, 3, "linear"),
    ([5, 3], 7, 5, 1, "linear"),
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-4), (torch.float16, 2e-2), (torch.bfloat16, 1e-1)])
def test_conv2d_vs_torch(case, dtype, tol):
    from ptlflow_b200 import _lib

    ops = _ops()
    chans, cout, kh, kw, epi = case
    b, h, w = 2, 11, 13
    cin = sum(chans)
    conv = torch.nn.Conv2d(cin, cout, (kh, kw), padding=(kh // 2, kw // 2))
    conv.weight.data = torch.from_numpy(synth.synth_normal("cv/w", tuple(conv.weight.shape), 3, scale=1.0 / math.sqrt(cin * kh * kw)))
    conv.bias.data = torch.from_numpy(synth.synth_normal("cv/b", (cout,), 3, scale=0.1))
    xs = [torch.from_numpy(synth.synth_normal(f"cv/x{i}", (b, c, h, w), 3)) for i, c in enumerate(chans)]
    xs_q = [x.to(dtype).float() for x in xs]  # the kernel sees storage-rounded inputs
    wq = conv.weight.data.to(dtype).float()
    ref = F.conv2d(torch.cat(xs_q, 1), wq, conv.bias.data, padding=(kh // 2, kw // 2))
    if epi == "relu":
        ref = torch.relu(ref)
    packed = ops.PackedConv([conv], dtype, DEV)
    out = torch.empty((b, h, w, cout + 3), dtype=dtype, device=DEV).fill_(7.0)
    ops.conv2d([_nhwc(x, dtype) for x in xs], packed, out, _lib.EPI_RELU if epi == "relu" else _lib.EPI_LINEAR, out_offset=1, impl=1)
    got = out[..., 1 : 1 + cout].permute(0, 3, 1, 2).float().cpu()
    assert (got - ref).abs().max().item() < tol
    assert (out[..., 0] == 7).all() and (out[..., 1 + cout :] == 7).all(), "wrote outside its channel window"


# ------------------------------------------------------------------------------------------
# a6-a9: update blocks against the reference's own modules (golden)
# ------------------------------------------------------------------------------------------
def _update_case(variant):
    recipe, g = load_golden(f"op_update_{variant}")
    hd, cd, rr, seed = recipe["hidden"], recipe["context"], recipe["radius"], recipe["seed"]
    bb, hh, ww = recipe["b"], recipe["h"], recipe["w"]
    planes = 4 * (2 * rr + 1) ** 2
    net = torch.tanh(torch.from_numpy(synth.synth_normal("ub/net", (bb, hd, hh, ww), seed)))
    inp = torch.relu(torch.from_numpy(synth.synth_normal("ub/inp", (bb, cd, hh, ww), seed)))
    corr = torch.from_numpy(synth.synth_normal("ub/corr", (bb, planes, hh, ww), seed))
    flow = torch.from_numpy(synth.synth_normal("ub/flow", (bb, 2, hh, ww), seed, scale=3.0))
    return recipe, g, net, inp, corr, flow


@pytest.mark.parametrize("variant", ["raft", "raft_small"])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 5e-5), (torch.float16, 1e-2)])
def test_update_block_vs_reference_vectors(variant, dtype, tol):
    import ptlflow_b200 as pb
    from ptlflow_b200.engine import RaftEngine

    recipe, g, net, inp, corr, flow = _update_case(variant)
    model = pb.get_model(variant)
    shapes = {k: v for k, v in O.state_dict_shapes(variant).items() if k.startswith("update_block.")}
    sd = synth.synth_state_dict(shapes, recipe["seed"])
    model.update_block.load_state_dict({k[len("update_block."):]: v for k, v in sd.items()})
    eng = RaftEngine(model.update_block.to(DEV), model._variant, model.hidden_dim, model.context_dim, 4, recipe["radius"], dtype, torch.device(DEV), impl=1)
    b, _, h, w = net.shape
    coords = (O.coords_grid(b, h, w) + flow).permute(0, 2, 3, 1).contiguous().to(DEV)
    net_d, inp_d = _nhwc(net, dtype), _nhwc(inp, dtype)
    mask = eng.update_iter(net_d, inp_d, coords, corr=_nhwc(corr, dtype), want_mask=True)
    delta = (coords.cpu() - (O.coords_grid(b, h, w) + flow).permute(0, 2, 3, 1)).permute(0, 3, 1, 2)
    assert np.abs(net_d.float().cpu().permute(0, 3, 1, 2).numpy() - g["net"]).max() < tol
    assert np.abs(delta.numpy() - g["delta"]).max() < tol
    if variant == "raft":
        assert np.abs(mask.float().cpu().permute(0, 3, 1, 2).numpy() - g["mask"]).max() < tol


# ------------------------------------------------------------------------------------------
# a10
# ------------------------------------------------------------------------------------------
def test_upsamplers_vs_reference_vectors():
    ops = _ops()
    recipe, g = load_golden("op_upsample")
    flow = torch.from_numpy(synth.synth_normal("up/flow", (2, 2, 7, 10), recipe["seed"], scale=3.0))
    mask = torch.from_numpy(synth.synth_normal("up/mask", (2, 576, 7, 10), recipe["seed"], scale=2.0))
    coords = (O.coords_grid(2, 7, 10) + flow).permute(0, 2, 3, 1).contiguous().to(DEV)
    up, small = ops.convex_upsample(coords, _nhwc(mask))
    assert np.abs(up.cpu().numpy() - g["convex"]).max() < 3e-5
    assert (small.cpu() - flow).abs().max().item() < 1e-5
    up8, _ = ops.upflow8(coords)
    assert np.abs(up8.cpu().numpy() - g["upflow8"]).max() < 3e-5
    # un-padded window == crop of the full result (the fused path writes rows 2..53 of 56 directly)
    upw, _ = ops.convex_upsample(coords, _nhwc(mask), out_hw=(52, 75), pad=(2, 3))
    assert torch.equal(upw, up[:, :, 2:54, 3:78])


# ------------------------------------------------------------------------------------------
# size-independent properties at BASELINE.json config-2 feature size (55x128, C=256)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_full_size_properties(dtype):
    ops = _ops()
    b, h, w, c, r, L = 1, 55, 128, 256, 4, 4
    g = torch.Generator(device="cpu").manual_seed(0)
    f1 = torch.randn(b, h, w, c, generator=g).to(DEV, dtype)
    f2 = torch.randn(b, h, w, c, generator=g).to(DEV, dtype)
    pyr = ops.corr_volume_build(f1, f2, L)
    assert [tuple(p.shape) for p in pyr] == [(7040, 55, 128), (7040, 27, 64), (7040, 13, 32), (7040, 6, 16)]
    tol = 1e-4 if dtype == torch.float32 else 3e-2
    # (1) zero-flow lookup: centre tap of level 0 is the diagonal <f1(q), f2(q)> / sqrt(C)
    coords = ops.init_coords(b, h, w, DEV)
    look = ops.corr_lookup(pyr, coords, r, (h, w), nchw=True, out_dtype=torch.float32)
    diag = (f1.float() * f2.float()).sum(-1) / math.sqrt(c)
    centre = look[:, (2 * r + 1) * r + r]
    assert (centre - diag).abs().max().item() < tol
    # (2) integer shift of the query coordinates permutes window entries: sample(x+1, i) == sample(x, i+1)
    shifted = coords.clone()
    shifted[..., 0] += 1.0
    look_s = ops.corr_lookup(pyr, shifted, r, (h, w), nchw=True, out_dtype=torch.float32)
    K = 2 * r + 1
    a = look_s[:, : K * K].reshape(b, K, K, h, w)[:, :-1]
    bb = look[:, : K * K].reshape(b, K, K, h, w)[:, 1:]
    assert (a - bb).abs().max().item() < 1e-6
    # (3) pooling conserves the mean on the even-cropped region
    lvl0, lvl1 = pyr[0].float(), pyr[1].float()
    assert (lvl0[:, :54, :].reshape(7040, 27, 2, 64, 2).mean(dim=(2, 4)) - lvl1).abs().max().item() < (1e-5 if dtype == torch.float32 else 2e-3)
    # (4) linearity in fmap1 (fp32 only): vol(2 f1) == 2 vol(f1)
    if dtype == torch.float32:
        pyr2 = ops.corr_volume_build(2 * f1, f2, 1)
        assert (pyr2[0] - 2 * pyr[0]).abs().max().item() < 1e-4
    # (5) on-the-fly == materialised
    fpyr = ops.feature_pyramid(f2, L)
    noisy = coords + 3.0 * torch.randn(coords.shape, generator=g).to(DEV)
    a = ops.corr_lookup(pyr, noisy, r, (h, w), out_dtype=torch.float32)
    bb = ops.corr_lookup_onthefly(f1, fpyr, noisy, r, out_dtype=torch.float32)
    assert (a - bb).abs().max().item() < (2e-4 if dtype == torch.float32 else 5e-2)


# ------------------------------------------------------------------------------------------
# encoder-side kernels (SURVEY 8(f) rank 1, first step)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(37, 50), (128, 160), (436, 1024)])
def test_preprocess_frames_vs_oracle(h, w):
    from ptlflow_b200.utils.utils import InputPadder

    ops = _ops()
    img = torch.from_numpy(synth.synth_images(2, h, w, 3, "noise"))
    ref, pads = O.preprocess(img)  # [B,2,3,Hp,Wp]
    padder = InputPadder(img.shape, stride=8)
    out = ops.preprocess_frames(img.to(DEV), padder.tgt_size, padder.pad_top_left)
    assert out.shape == (4, ref.shape[-2], ref.shape[-1], 3)
    got = out.permute(0, 3, 1, 2).cpu()
    assert torch.equal(got[:2], ref[:, 0]) and torch.equal(got[2:], ref[:, 1])
    out4 = ops.preprocess_frames(img.to(DEV), padder.tgt_size, padder.pad_top_left, out_channels=4)  # 8-byte pixels for conv1
    assert out4.shape[-1] == 4 and torch.equal(out4[..., :3], out) and not out4[..., 3].any()


@pytest.mark.parametrize("c", [64, 96, 128, 24, 8])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.float16, 4e-3)])
def test_instance_norm_act_vs_torch(c, dtype, tol):
    ops = _ops()
    b, h, w = 3, 19, 27
    x = torch.from_numpy(synth.synth_normal("in/x", (b, c, h, w), 1, scale=2.0)) + 0.7
    res = torch.relu(torch.from_numpy(synth.synth_normal("in/r", (b, c, h, w), 2)))
    xq, rq = x.to(dtype).float(), res.to(dtype).float()
    base = F.instance_norm(xq, eps=1e-5)
    xd, rd = _nhwc(x, dtype), _nhwc(res, dtype)
    y = ops.instance_norm_act(xd, relu=True)
    assert (y.permute(0, 3, 1, 2).float().cpu() - torch.relu(base)).abs().max().item() < tol
    y = ops.instance_norm_act(xd, relu=False)
    assert (y.permute(0, 3, 1, 2).float().cpu() - base).abs().max().item() < tol
    y = ops.instance_norm_act(xd, relu=True, residual=rd)
    assert (y.permute(0, 3, 1, 2).float().cpu() - torch.relu(rq + torch.relu(base))).abs().max().item() < 2 * tol
    bias = torch.from_numpy(synth.synth_normal("in/b", (c,), 3, scale=0.3))
    y = ops.bias_act(xd, bias.to(DEV), relu=True, residual=rd)
    assert (y.permute(0, 3, 1, 2).float().cpu() - torch.relu(rq + torch.relu(xq + bias.view(1, -1, 1, 1)))).abs().max().item() < 2 * tol
    y = ops.bias_act(xd, bias.to(DEV), relu=False)
    assert (y.permute(0, 3, 1, 2).float().cpu() - (xq + bias.view(1, -1, 1, 1))).abs().max().item() < 2 * tol


@pytest.mark.parametrize("variant", ["raft", "raft_small"])
def test_encoders_vs_oracle_fp32(variant):
    import ptlflow_b200 as pb

    small = variant == "raft_small"
    sd = synth.synth_state_dict(O.state_dict_shapes(variant), 3)
    model = pb.get_model(variant)
    model.load_state_dict(sd)
    model = model.eval().to(DEV)
    img = torch.from_numpy(synth.synth_images(2, 72, 104, 4, "smooth"))
    x, _ = O.preprocess(img)
    frames = x.transpose(0, 1).reshape(4, 3, 72, 104)  # frame-major
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        f = model.fnet.forward_pm(frames.permute(0, 2, 3, 1).contiguous().to(DEV))
        c = model.cnet.forward_pm(frames[:2].permute(0, 2, 3, 1).contiguous().to(DEV))
    fref = O.encoder(frames, sd, "fnet.", "instance", small)
    cref = O.encoder(frames[:2], sd, "cnet.", "none" if small else "batch", small)
    assert (f.permute(0, 3, 1, 2).cpu() - fref).abs().max().item() < 2e-4
    assert (c.permute(0, 3, 1, 2).cpu() - cref).abs().max().item() < 2e-4


# ------------------------------------------------------------------------------------------
# a13: GMA attention + aggregate (operator level, against the oracle)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.float16, 2e-2)])
@pytest.mark.parametrize("h,w", [(8, 16), (9, 13)])  # N = 128 (tensor path in f16) and N = 117 (SIMT fallback)
def test_gma_attention_and_aggregate_vs_oracle(dtype, tol, h, w):
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib
    from ptlflow_b200.engine import RaftEngine

    ops = _ops()
    b = 2
    sd = synth.synth_state_dict({k: v for k, v in O.state_dict_shapes("gma").items() if k.split(".")[0] in ("update_block", "att")}, 5)
    model = pb.get_model("gma")
    model.update_block.load_state_dict({k[len("update_block."):]: v for k, v in sd.items() if k.startswith("update_block.")})
    model.att.load_state_dict({k[len("att."):]: v for k, v in sd.items() if k.startswith("att.")})
    model.update_block.to(DEV), model.att.to(DEV)
    eng = RaftEngine(model.update_block, 2, 128, 128, 4, 4, dtype, torch.device(DEV), attention_module=model.att)
    inp = torch.relu(torch.from_numpy(synth.synth_normal("gma/inp", (b, 128, h, w), 6)))
    attn_ref = O.gma_attention(inp.to(dtype).float(), {k: v.to(dtype).float() for k, v in sd.items()})
    attn = model._attention(_nhwc(inp, dtype), eng)
    assert attn.shape == (b * h * w, h * w)
    assert (attn.float().cpu().view(b, h * w, h * w) - attn_ref).abs().max().item() < tol
    assert (attn.float().sum(-1) - 1).abs().max().item() < (1e-5 if dtype == torch.float32 else 5e-3)


@pytest.mark.parametrize("n,h,w", [(2, 48, 64), (1, 18, 1040), (3, 20, 1024), (1, 8, 8)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mode", ["instance", "bias_relu"])
def test_first_conv7x7s2_vs_torch(n, h, w, dtype, mode):
    """wgmma first convolution (overlapping-window operand descriptors) against F.conv2d on the same rounded
    inputs, fp32 accumulate; the instance-norm sums from its epilogue against torch sums of the fp32 result."""
    import torch.nn.functional as F

    ops = _ops()
    wt = torch.from_numpy(synth.synth_normal("fc/w", (64, 3, 7, 7), 5, scale=0.12))
    bias = torch.from_numpy(synth.synth_normal("fc/b", (64,), 5, scale=0.5))
    x3 = torch.from_numpy(synth.synth_normal("fc/x", (n, h, w, 3), 6, scale=0.6)).clamp(-1, 1)
    x4 = torch.zeros(n, h, w, 4)
    x4[..., :3] = x3
    xd = x4.to(DEV, dtype).contiguous()
    wq = wt.to(dtype).float()
    ref = F.conv2d(xd[..., :3].float().cpu().permute(0, 3, 1, 2), wq, None, stride=2, padding=3)  # [n,64,h/2,w/2]
    wpack = ops.pack_first_conv(wt, dtype).to(DEV)
    if mode == "instance":
        ws = ops.instance_norm_workspace((n, 0, 0, 64), DEV)
        out = ops.first_conv7x7s2(xd, wpack, None, relu=False, stats_ws=ws)
        sums = ws[: n * 64 * 2].view(n, 64, 2).cpu()
        assert torch.allclose(sums[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-3, atol=2e-2 * ref[0, 0].numel() ** 0.5)
        assert torch.allclose(sums[..., 1], (ref.double() ** 2).sum(dim=(2, 3)), rtol=2e-3, atol=1e-2)
    else:
        ref = torch.relu(ref + bias.view(1, -1, 1, 1))
        out = ops.first_conv7x7s2(xd, wpack, bias.to(DEV), relu=True)
    got = out.float().cpu().permute(0, 3, 1, 2)
    assert got.shape == ref.shape
    tol = 6e-3 if dtype == torch.float16 else 4e-2
    err = (got - ref).abs().max().item()
    assert err < tol * max(1.0, ref.abs().max().item()), f"max-abs error {err}"


@pytest.mark.parametrize("b,h,w", [(2, 11, 21), (1, 55, 128), (1, 5, 300)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_flow_conv7x7_vs_torch(b, h, w, dtype):
    """Tensor-core convf1 (hi/lo split of the fp32 flow) == fp32 flow x storage-type weights, fp32 accumulate."""
    import torch.nn.functional as F

    ops = _ops()
    wt = torch.from_numpy(synth.synth_normal("fl/w", (128, 2, 7, 7), 7, scale=0.1))
    bias = torch.from_numpy(synth.synth_normal("fl/b", (128,), 7, scale=0.3))
    flow = torch.from_numpy(synth.synth_normal("fl/x", (b, h, w, 2), 8, scale=25.0))
    ref = torch.relu(F.conv2d(flow.permute(0, 3, 1, 2), wt.to(dtype).float(), bias, padding=3))  # [b,128,h,w]
    out = torch.full((b, h, w, 160), 7.0, dtype=dtype, device=DEV)
    ops.flow_conv7x7(flow.to(DEV), ops.pack_flow_conv(wt, dtype).to(DEV), bias.to(DEV), out, out_offset=16)
    got = out[..., 16:144].float().cpu().permute(0, 3, 1, 2)
    assert (out[..., :16] == 7).all() and (out[..., 144:] == 7).all()
    eps = 1e-3 if dtype == torch.float16 else 8e-3
    err = ((got - ref).abs() / (1.0 + ref.abs())).max().item()
    assert err < 2 * eps, f"relative error {err}"


@pytest.mark.parametrize("b,h,w,scale", [(2, 16, 24, 3.0), (1, 55, 128, 8.0), (1, 9, 11, 40.0)])
def test_forward_interpolate_vs_scipy(b, h, w, scale):
    """Device warm start == the reference's scipy griddata(nearest) forward_interpolate (utils/external/raft.py:155-185);
    the only admissible differences are exact distance ties."""
    from ptlflow_b200.utils.warm_start import forward_interpolate_batch

    flow = torch.from_numpy(synth.synth_normal("fi/flow", (b, 2, h, w), 9, scale=scale))
    ref = forward_interpolate_batch(flow)  # host tensors: scipy restatement of the reference
    got = forward_interpolate_batch(flow.to(DEV)).cpu()
    assert got.shape == ref.shape
    mismatch = ((got - ref).abs().amax(dim=1) > 0).float().mean().item()
    assert mismatch < 2e-3, f"{mismatch:.4f} of the pixels differ from scipy's nearest neighbour"
    assert torch.equal(forward_interpolate_batch(torch.full((1, 2, 6, 7), 1000.0, device=DEV)).cpu(), torch.zeros(1, 2, 6, 7))  # nothing lands inside


def test_forward_interpolate_vs_reference_vector():
    """pfb_forward_interpolate against the vector written by the reference's own forward_interpolate_batch."""
    from helpers import load_golden
    from ptlflow_b200.utils.warm_start import forward_interpolate_batch

    recipe, g = load_golden("op_forward_interpolate")
    flow = torch.from_numpy(synth.synth_normal("ws/flow", (recipe["b"], 2, recipe["h"], recipe["w"]), recipe["seed"], scale=recipe["scale"]))
    got = forward_interpolate_batch(flow.to(DEV)).cpu().numpy()
    mismatch = (np.abs(got - g["out"]).max(axis=1) > 0).mean()
    assert mismatch < 2e-3, f"{mismatch:.4f} of the pixels differ from the reference (only exact distance ties may)"
