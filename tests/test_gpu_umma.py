"""GPU parity tests for the wgmma / TMA kernels (f16, bf16): the tensor-core correlation-volume GEMM
with its fused pyramid epilogue, the implicit-GEMM convolution with every fused epilogue, and the two
dedicated small convolutions.  Checkers: torch fp32 on storage-rounded inputs, and the SIMT kernels
(impl=1) of the same library, which tests/test_gpu_ops.py pins to the reference vectors."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _nhwc(x, dtype):
    return x.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)


def _q(x, dtype):
    return x.to(dtype).float()


# ------------------------------------------------------------------------------------------
# correlation volume + pyramid
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,h,w,c,levels", [(2, 17, 24, 64, 4), (1, 16, 16, 128, 3), (1, 55, 128, 256, 4), (3, 9, 50, 192, 2), (1, 8, 16, 256, 1)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_corr_volume_umma_vs_simt_and_torch(b, h, w, c, levels, dtype):
    from ptlflow_b200 import ops

    f1 = torch.from_numpy(synth.synth_normal("u/f1", (b, c, h, w), 1))
    f2 = torch.from_numpy(synth.synth_normal("u/f2", (b, c, h, w), 1))
    a, bb = _nhwc(f1, dtype), _nhwc(f2, dtype)
    tc = ops.corr_volume_build(a, bb, levels, impl=2)
    simt = ops.corr_volume_build(a, bb, levels, impl=1)
    ref = O.corr_pyramid(O.corr_volume(_q(f1, dtype), _q(f2, dtype)), levels)
    ulp = 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7
    for lvl, (t, s, r) in enumerate(zip(tc, simt, ref)):
        assert t.shape == s.shape
        scale = max(1.0, r.abs().max().item())
        # same inputs, fp32 accumulation in a different order: at most a rounding flip of the stored value
        assert (t.float() - s.float()).abs().max().item() <= 2.5 * ulp * scale, f"level {lvl}"
        assert (t.float().cpu() - r[:, 0]).abs().max().item() <= 4 * ulp * scale, f"level {lvl} vs torch"


# ------------------------------------------------------------------------------------------
# implicit-GEMM convolution
# ------------------------------------------------------------------------------------------
def _make_conv(cin, cout, kh, kw, seed):
    conv = torch.nn.Conv2d(cin, cout, (kh, kw), padding=(kh // 2, kw // 2))
    conv.weight.data = torch.from_numpy(synth.synth_normal(f"uc/w{seed}", tuple(conv.weight.shape), seed, scale=1.0 / math.sqrt(cin * kh * kw)))
    conv.bias.data = torch.from_numpy(synth.synth_normal(f"uc/b{seed}", (cout,), seed, scale=0.1))
    return conv


UMMA_CONV_CASES = [
    # name, source channel counts, Cout, KH, KW
    ("convc1", [324], 256, 1, 1),
    ("convc2", [256], 192, 3, 3),
    ("convf2", [128], 64, 3, 3),
    ("mask2", [256], 576, 1, 1),
    ("flow1", [128], 256, 3, 3),
    ("three_src_1x5", [128, 128, 128], 128, 1, 5),
    ("three_src_5x1", [128, 128, 128], 128, 5, 1),
]


@pytest.mark.parametrize("case", UMMA_CONV_CASES, ids=[c[0] for c in UMMA_CONV_CASES])
@pytest.mark.parametrize("b,h,w", [(2, 11, 21), (1, 16, 32), (1, 5, 128), (2, 3, 200)])  # W >= 128: row tiles + halo reuse
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_conv_umma_relu_linear(case, b, h, w, dtype):
    from ptlflow_b200 import _lib, ops

    name, chans, cout, kh, kw = case
    conv = _make_conv(sum(chans), cout, kh, kw, 11)
    xs = [torch.from_numpy(synth.synth_normal(f"uc/x{i}", (b, c, h, w), 12)) for i, c in enumerate(chans)]
    ref = F.conv2d(torch.cat([_q(x, dtype) for x in xs], 1), _q(conv.weight.data, dtype), conv.bias.data, padding=(kh // 2, kw // 2))
    packed = ops.PackedConv([conv], dtype, DEV, src_channels=chans)
    assert packed.weight_k is not None
    srcs = []
    for x, c in zip(xs, chans):
        t = _nhwc(x, dtype)
        if c % 64:  # storage padded to a 16-byte multiple; pad columns hold garbage on purpose: the TMA box
            pad = torch.full((b, h, w, (c + 63) // 64 * 64 - c), float("nan"), dtype=dtype, device=DEV)  # must zero-fill them
            t = torch.cat([t, pad], -1).contiguous()
            srcs.append((t, c, 0))
        else:
            srcs.append(t)
    for epi, fn, scale in ((_lib.EPI_RELU, torch.relu, 1.0), (_lib.EPI_LINEAR, lambda v: 0.25 * v, 0.25)):
        out = torch.full((b, h, w, cout + 8), 7.0, dtype=dtype, device=DEV)
        ops.conv2d(srcs, packed, out, epi, out_offset=8, scale=scale, impl=2)
        got = out[..., 8:].permute(0, 3, 1, 2).float().cpu()
        tol = (2e-3 if dtype == torch.float16 else 1.6e-2) * max(1.0, ref.abs().max().item())
        assert (got - fn(ref)).abs().max().item() < tol, name
        assert (out[..., :8] == 7).all()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("kh,kw", [(1, 5), (5, 1)])
@pytest.mark.parametrize("h,w", [(13, 19), (6, 128), (23, 130)])
def test_conv_umma_gru_epilogues(dtype, kh, kw, h, w):
    """z|r fused GEMM (N = 256) + q GEMM with the gate arithmetic of update.py:58-73 in the epilogue."""
    from ptlflow_b200 import _lib, ops

    b, hd = 2, 128
    convz, convr, convq = (_make_conv(384, 128, kh, kw, s) for s in (21, 22, 23))
    net = torch.tanh(torch.from_numpy(synth.synth_normal("g/net", (b, hd, h, w), 3)))
    inp = torch.relu(torch.from_numpy(synth.synth_normal("g/inp", (b, 128, h, w), 3)))
    mot = torch.relu(torch.from_numpy(synth.synth_normal("g/mot", (b, 128, h, w), 3)))
    qd = lambda t: _q(t, dtype)  # noqa: E731
    pad = (kh // 2, kw // 2)
    hx = torch.cat([qd(net), qd(inp), qd(mot)], 1)
    z = torch.sigmoid(F.conv2d(hx, qd(convz.weight.data), convz.bias.data, padding=pad))
    r = torch.sigmoid(F.conv2d(hx, qd(convr.weight.data), convr.bias.data, padding=pad))
    rh = qd(r * qd(net))
    qv = torch.tanh(F.conv2d(torch.cat([rh, qd(inp), qd(mot)], 1), qd(convq.weight.data), convq.bias.data, padding=pad))
    hnew = (1 - qd(z)) * qd(net) + qd(z) * qv

    pzr = ops.PackedConv([convz, convr], dtype, DEV, src_channels=[128, 128, 128])
    pq = ops.PackedConv([convq], dtype, DEV, src_channels=[128, 128, 128])
    net_d, inp_d, mot_d = _nhwc(net, dtype), _nhwc(inp, dtype), _nhwc(mot, dtype)
    z_d = torch.empty_like(net_d)
    rh_d = torch.empty_like(net_d)
    ops.conv2d([net_d, inp_d, mot_d], pzr, rh_d, _lib.EPI_GRU_ZR, aux_h=net_d, aux_z=z_d, hidden=hd, impl=2)
    tol = 3e-3 if dtype == torch.float16 else 2e-2
    assert (z_d.permute(0, 3, 1, 2).float().cpu() - z).abs().max().item() < tol
    assert (rh_d.permute(0, 3, 1, 2).float().cpu() - r * qd(net)).abs().max().item() < tol
    ops.conv2d([rh_d, inp_d, mot_d], pq, net_d, _lib.EPI_GRU_Q, aux_h=net_d, aux_z=z_d, hidden=hd, impl=2)
    assert (net_d.permute(0, 3, 1, 2).float().cpu() - hnew).abs().max().item() < 3 * tol


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_conv_umma_append_flow_and_special_kernels(dtype):
    from ptlflow_b200 import _lib, ops

    b, h, w = 2, 11, 21
    qd = lambda t: _q(t, dtype)  # noqa: E731
    tol = 3e-3 if dtype == torch.float16 else 2e-2
    flow = torch.from_numpy(synth.synth_normal("s/flow", (b, 2, h, w), 4, scale=3.0))
    flow_d = flow.permute(0, 2, 3, 1).contiguous().to(DEV)
    # motion-encoder output conv: 126 channels + the two flow columns (update.py:111-112)
    conv = _make_conv(256, 126, 3, 3, 31)
    x = torch.relu(torch.from_numpy(synth.synth_normal("s/x", (b, 256, h, w), 4)))
    ref = torch.cat([torch.relu(F.conv2d(qd(x), qd(conv.weight.data), conv.bias.data, padding=1)), flow], 1)
    out = torch.zeros((b, h, w, 128), dtype=dtype, device=DEV)
    ops.conv2d([_nhwc(x, dtype)], ops.PackedConv([conv], dtype, DEV, src_channels=[256]), out, _lib.EPI_RELU_APPEND_FLOW, flow=flow_d, impl=2)
    assert (out.permute(0, 3, 1, 2).float().cpu() - ref).abs().max().item() < max(tol, 3.0 * 2 ** (-10 if dtype == torch.float16 else -7) * 4)
    # 7x7 conv on the fp32 flow (dedicated kernel), Cout 128 and 64
    for cout in (128, 64):
        c7 = _make_conv(2, cout, 7, 7, 32)
        ref7 = torch.relu(F.conv2d(flow, qd(c7.weight.data), c7.bias.data, padding=3))
        o7 = torch.zeros((b, h, w, cout), dtype=dtype, device=DEV)
        ops.conv2d([flow_d], ops.PackedConv([c7], dtype, DEV), o7, _lib.EPI_RELU, impl=0)
        assert (o7.permute(0, 3, 1, 2).float().cpu() - ref7).abs().max().item() < tol * max(1.0, ref7.abs().max().item())
    # flow head conv2 (256 -> 2) fused with the coordinate update (dedicated kernel)
    c2 = _make_conv(256, 2, 3, 3, 33)
    delta = F.conv2d(qd(x), qd(c2.weight.data), c2.bias.data, padding=1)
    coords0 = O.coords_grid(b, h, w) + flow
    coords = coords0.permute(0, 2, 3, 1).contiguous().to(DEV)
    fout = torch.zeros((b, h, w, 2), dtype=torch.float32, device=DEV)
    ops.conv2d([_nhwc(x, dtype)], ops.PackedConv([c2], dtype, DEV, src_channels=[256]), fout, _lib.EPI_FLOW, coords=coords, impl=0)
    assert (coords.permute(0, 3, 1, 2).cpu() - (coords0 + delta)).abs().max().item() < 2e-3
    assert (fout.permute(0, 3, 1, 2).cpu() - (flow + delta)).abs().max().item() < 2e-3


def test_update_block_tcgen05_vs_simt():
    """One full BasicUpdateBlock evaluation: auto (wgmma + dedicated kernels) against SIMT, f16."""
    import ptlflow_b200 as pb
    from ptlflow_b200.engine import RaftEngine

    b, h, w = 2, 20, 35
    model = pb.get_model("raft")
    sd = synth.synth_state_dict({k: v for k, v in O.state_dict_shapes("raft").items() if k.startswith("update_block.")}, 9)
    model.update_block.load_state_dict({k[len("update_block."):]: v for k, v in sd.items()})
    model.update_block.to(DEV)
    f1 = torch.from_numpy(synth.synth_normal("ub2/f1", (b, 256, h, w), 2))
    f2 = torch.from_numpy(synth.synth_normal("ub2/f2", (b, 256, h, w), 2))
    net = torch.tanh(torch.from_numpy(synth.synth_normal("ub2/net", (b, 128, h, w), 2)))
    inp = torch.relu(torch.from_numpy(synth.synth_normal("ub2/inp", (b, 128, h, w), 2)))
    flow = torch.from_numpy(synth.synth_normal("ub2/flow", (b, 2, h, w), 2, scale=2.0))
    from ptlflow_b200 import ops

    res = []
    for impl in (1, 0):
        eng = RaftEngine(model.update_block, 0, 128, 128, 4, 4, torch.float16, torch.device(DEV), impl=impl)
        pyr = ops.corr_volume_build(_nhwc(f1, torch.float16), _nhwc(f2, torch.float16), 4, impl=impl)
        coords = (O.coords_grid(b, h, w) + flow).permute(0, 2, 3, 1).contiguous().to(DEV)
        net_d = _nhwc(net, torch.float16)
        mask = eng.update_iter(net_d, _nhwc(inp, torch.float16), coords, pyramid=pyr, want_mask=True)
        res.append((net_d.float().cpu(), coords.cpu(), mask.float().cpu()))
    for a, c, nm, tol in zip(res[0], res[1], ("net", "coords", "mask"), (6e-3, 6e-3, 2e-2)):
        assert (a - c).abs().max().item() < tol, nm
