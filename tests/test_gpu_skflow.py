"""GPU: SKFlow against the oracle and the reference vectors.

Kernels: the fused depthwise convolution + residual + GELU against F.conv2d(groups=C) for several kernel sizes, channel counts,
grids smaller than the kernel and strided inputs in fp32 / f16 / bf16; the GELU, residual-GELU and linear-append-flow epilogues
of the convolution on the wgmma and the SIMT kernels.  Update block: one iteration against skflow_oracle.update_block on the
tensor path and with kernel_impl = 1.  End to end: the e2e_skflow_* reference vectors in fp32, f16 / bf16 against them, the
config-3 image size in half precision against the fp32 oracle, CUDA-graph replay against the eager forward, and the grid limit
of the positional attention modes.
"""
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import skflow_oracle as SO
from helpers import load_golden
from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = os.environ.get("PFB_PARITY_REPORT")  # optional: one JSON line of measured errors per check
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
TOL = {torch.float32: 2e-5, torch.float16: 1e-2, torch.bfloat16: 6e-2}


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

    model = pb.get_model("skflow", args=Namespace(model=Namespace(**kwargs)))
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    model = model.eval().to(DEV)
    if dtype != torch.float32:
        model = model.to(dtype)
    model.kernel_impl = impl
    return model


# --------------------------------------------------------------------------------------
# depthwise kernel
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C", [128, 256, 324, 512])
@pytest.mark.parametrize("k", [1, 3, 7, 15])
def test_depthwise_vs_conv2d(k, C, dtype):
    from ptlflow_b200 import ops

    w = _gen(f"dw/w{k}", (C, 1, k, k), 1, scale=1.0 / k)
    b = _gen(f"dw/b{k}", (C,), 2, scale=0.1)
    wt = w.reshape(C, k * k).t().contiguous().to(DEV)
    for bsz, h, wd, pad in ((2, 6, 9, 0), (1, 17, 23, 8)):  # 6x9: smaller than 15x15; the second one reads a strided slice
        x = _gen(f"dw/x{h}", (bsz, C, h, wd), 3).to(dtype).float()
        ref = SO.gelu(x + F.conv2d(x, w, b, padding=k // 2, groups=C))
        src = torch.zeros((bsz, h, wd, C + 2 * pad), dtype=dtype, device=DEV)
        src[..., pad:pad + C] = x.permute(0, 2, 3, 1).to(DEV, dtype)
        out = ops.depthwise_conv_gelu(src, wt, b.to(DEV), k, channels=C, in_offset=pad)
        torch.cuda.synchronize()
        err = (out.float().cpu().permute(0, 3, 1, 2) - ref).abs().max().item()
        _report(test="depthwise", k=k, C=C, dtype=str(dtype), grid=f"{h}x{wd}", err=err)
        assert err < TOL[dtype] * max(1.0, ref.abs().max().item()), (h, wd, err)


def test_depthwise_k31_into_a_strided_output():
    from ptlflow_b200 import ops

    C, k = 64, 31
    w, b = _gen("dw/w31", (C, 1, k, k), 1, scale=1.0 / k), _gen("dw/b31", (C,), 2, scale=0.1)
    x = _gen("dw/x31", (1, C, 20, 40), 3)
    ref = SO.gelu(x + F.conv2d(x, w, b, padding=k // 2, groups=C))
    out = torch.full((1, 20, 40, 96), 7.0, device=DEV)
    ops.depthwise_conv_gelu(x.permute(0, 2, 3, 1).contiguous().to(DEV), w.reshape(C, -1).t().contiguous().to(DEV), b.to(DEV), k,
                            out=out, out_offset=16)
    torch.cuda.synchronize()
    assert (out[..., 16:80].cpu().permute(0, 3, 1, 2) - ref).abs().max().item() < 2e-5
    assert (out[..., :16] == 7).all() and (out[..., 80:] == 7).all()


# --------------------------------------------------------------------------------------
# convolution epilogues
# --------------------------------------------------------------------------------------
class _Conv:
    def __init__(self, cout, cin, seed):
        self.weight = _gen(f"epi/w{cout}x{cin}", (cout, cin, 1, 1), seed, scale=cin ** -0.5)
        self.bias = _gen(f"epi/b{cout}", (cout,), seed, scale=0.1)


EPI_CASES = [(d, i) for d in DTYPES for i in ((0, 1) if d != torch.float32 else (0,))]


@pytest.mark.parametrize("dtype,impl", EPI_CASES, ids=[f"{str(d)[6:]}-impl{i}" for d, i in EPI_CASES])
def test_new_epilogues(dtype, impl):
    """GELU, RESIDUAL_GELU (strided residual, with and without the per-channel step) and LINEAR_APPEND_FLOW; impl 0 on f16 / bf16
    is the wgmma kernel (impl 2 would raise if it were not), impl 1 the SIMT kernel."""
    from ptlflow_b200 import _lib, ops

    b, h, w, cin, cout = 2, 9, 20, 192, 256
    conv = _Conv(cout, cin, 4)
    pc = ops.PackedConv([conv], dtype, DEV, src_channels=[cin])
    x = _gen("epi/x", (b, h, w, cin), 5).to(dtype)
    acc = (x.float() @ conv.weight[:, :, 0, 0].t() + conv.bias)  # [b,h,w,cout]
    xd = x.to(DEV)
    run_impl = 2 if (dtype != torch.float32 and impl == 0) else impl

    out = torch.empty((b, h, w, cout), dtype=dtype, device=DEV)
    ops.conv2d([xd], pc, out, epilogue=_lib.EPI_GELU, impl=run_impl)
    errs = {"gelu": (out.float().cpu() - SO.gelu(acc)).abs().max().item()}

    res = _gen("epi/res", (b, h, w, cout + 64), 6).to(dtype)
    pw_, pb_ = _gen("epi/pw", (cout,), 7, scale=0.5), _gen("epi/pb", (cout,), 8, scale=0.1)
    y = SO.gelu(res[..., 32:32 + cout].float() + acc)
    for post in (False, True):
        out = torch.empty((b, h, w, cout), dtype=dtype, device=DEV)
        ops.conv2d([xd], pc, out, epilogue=_lib.EPI_RESIDUAL_GELU, impl=run_impl, residual=(res.to(DEV), 32),
                   post_w=pw_.to(DEV) if post else None, post_b=pb_.to(DEV) if post else None)
        ref = SO.gelu(y * (1 + pw_) + pb_) if post else y
        errs[f"residual_gelu_post{int(post)}"] = (out.float().cpu() - ref).abs().max().item()

    conv126 = _Conv(126, cin, 9)
    pc126 = ops.PackedConv([conv126], dtype, DEV, src_channels=[cin])
    flow = _gen("epi/flow", (b, h, w, 2), 10, scale=3.0).to(DEV)
    out = torch.zeros((b, h, w, 512), dtype=dtype, device=DEV)
    ops.conv2d([xd], pc126, out, epilogue=_lib.EPI_LINEAR_APPEND_FLOW, out_offset=256, flow=flow, impl=run_impl)
    ref = torch.cat([x.float() @ conv126.weight[:, :, 0, 0].t() + conv126.bias, flow.cpu().to(dtype).float()], -1)
    errs["linear_append_flow"] = (out[..., 256:384].float().cpu() - ref).abs().max().item()
    assert (out[..., :256] == 0).all() and (out[..., 384:] == 0).all()
    torch.cuda.synchronize()
    _report(test="skflow_epilogues", dtype=str(dtype), impl=impl, **errs)
    tol = {torch.float32: 1e-4, torch.float16: 1e-2, torch.bfloat16: 6e-2}[dtype]
    for name, e in errs.items():
        assert e < tol, (name, e)


# --------------------------------------------------------------------------------------
# one update iteration
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(9, 13), (8, 16)])  # N = 117 (SIMT aggregate in half precision, 9 < 15) and N = 128; 4 levels
@pytest.mark.parametrize("dtype,impl", [(torch.float32, 0), (torch.float16, 0), (torch.bfloat16, 0), (torch.float16, 1)])
def test_update_iteration_vs_oracle(dtype, impl, h, w):
    """One SKFlow update block (two heads, position_and_content) against skflow_oracle.update_block on the same storage-rounded
    inputs: new net, delta flow and the mask."""
    import ptlflow_b200 as pb
    from ptlflow_b200 import ops
    from ptlflow_b200.engine import SKFlowEngine

    b = 2 if h == 9 else 1
    sd, net, inp, corr, flow, attn = SO.op_iter_inputs(b, h, w)
    q = lambda t: t.to(dtype).float()  # noqa: E731
    sdq = {k: q(v) for k, v in sd.items()}
    net, inp, corr, flow = q(net), q(inp), q(corr), q(flow)
    attn = q(attn)
    n_ref, m_ref, d_ref = SO.update_block(net, inp, corr, flow, attn, sdq)
    model = pb.get_model("skflow", args=Namespace(model=Namespace(num_heads=2, position_and_content=True)))
    model.update_block.load_state_dict({k[len("update_block."):]: v for k, v in sd.items() if k.startswith("update_block.")})
    model.att.load_state_dict({k[len("att."):]: v for k, v in sd.items() if k.startswith("att.")}, strict=False)
    model.update_block.to(DEV, dtype), model.att.to(DEV, dtype)
    eng = SKFlowEngine(model.update_block, 3, 128, 128, 4, 4, dtype, torch.device(DEV), impl=impl, attention_module=model.att)
    coords0 = O.coords_grid(b, h, w)
    coords = ops.coords_to_pixel_major(coords0 + flow).to(DEV)
    net_d = net.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)
    corr_d = torch.zeros((b, h, w, eng.corr_stride), dtype=dtype, device=DEV)
    corr_d[..., :324] = corr.permute(0, 2, 3, 1).to(DEV, dtype)
    attn_d = attn.transpose(0, 1).reshape(2 * b * h * w, h * w).to(DEV, dtype).contiguous()
    with torch.no_grad():
        mask = eng.update_iter(net_d, inp.permute(0, 2, 3, 1).contiguous().to(DEV, dtype), coords, corr=corr_d, want_mask=True,
                               attention=attn_d)
    torch.cuda.synchronize()
    e_net = (net_d.float().cpu().permute(0, 3, 1, 2) - n_ref).abs().max().item()
    e_delta = ((coords.cpu().permute(0, 3, 1, 2) - coords0 - flow) - d_ref).abs().max().item()
    e_mask = (mask.float().cpu().permute(0, 3, 1, 2) - m_ref).abs().max().item()  # (the oracle's mask head includes the 0.25)
    _report(test="skflow_update_iter", case=f"{h}x{w}", dtype=str(dtype), impl=impl, err_net=e_net, err_delta=e_delta, err_mask=e_mask,
            scale_net=n_ref.abs().max().item())
    tol = 1e-4 if dtype == torch.float32 else (2e-2 if dtype == torch.float16 else 1.5e-1)
    assert e_net < tol * max(1.0, n_ref.abs().max().item()) and e_delta < tol and e_mask < tol, (e_net, e_delta, e_mask)


# --------------------------------------------------------------------------------------
# end to end
# --------------------------------------------------------------------------------------
def _run(model, img, recipe, dtype=torch.float32):
    with torch.no_grad():
        if recipe.get("warm"):
            first = model({"images": img.to(DEV, dtype)})
            return model({"images": img.to(DEV, dtype), "prev_preds": {"flow_small": first["flow_small"]}}), first
        return model({"images": img.to(DEV, dtype)}), None


@pytest.mark.parametrize("name", SO.E2E)
def test_fp32_matches_reference_vectors(name):
    recipe, g = load_golden(name)
    sd, img, kw = SO.e2e_inputs(recipe)
    model = _model(kw, sd)
    out, first = _run(model, img, recipe)
    out2, _ = _run(model, img, recipe)  # replays the captured CUDA graph(s)
    err = np.abs(out["flows"].cpu().numpy() - g["flows"]).max()
    err2 = np.abs(out2["flows"].cpu().numpy() - g["flows"]).max()
    err_small = np.abs(out["flow_small"].cpu().numpy() - g["flow_small"]).max()
    if first is not None:
        assert np.abs(first["flow_small"].cpu().numpy() - g["first_flow_small"]).max() < 1e-3
    _report(test="skflow_fp32_golden", case=name, err_flow=float(err), err_replay=float(err2), err_flow_small=float(err_small))
    assert out["flows"].shape == g["flows"].shape
    assert err < 1e-3 and err2 < 1e-3 and err_small < 1e-3, f"{name}: max-abs flow error {err} / replay {err2} / small {err_small}"


@pytest.mark.parametrize("name", [n for n in SO.E2E if n != "e2e_skflow_warm"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_against_fp32_reference(name, dtype):
    recipe, g = load_golden(name)
    sd, img, kw = SO.e2e_inputs(recipe)
    model = _model(kw, sd, dtype)
    out, _ = _run(model, img, recipe, dtype)
    d = np.abs(out["flows_fp32"].cpu().numpy() - g["flows"])
    _report(test="skflow_half_vs_fp32_ref", case=name, dtype=str(dtype), err_flow=float(d.max()), mean_err=float(d.mean()))
    bound, mean_bound = (4e-2, 1e-2) if dtype == torch.float16 else (3e-1, 6e-2)
    assert d.max() < bound and d.mean() < mean_bound, f"{name} {dtype}: max-abs {d.max()} mean-abs {d.mean()}"


@pytest.mark.parametrize("dtype,gate_max,gate_mean", [(torch.bfloat16, 5e-1, 1e-1), (torch.float16, 8e-2, 2.5e-2)])
def test_config3_size_against_fp32_oracle(dtype, gate_max, gate_mean):
    """BASELINE config 3 image size (436x1024 -> 55x128 grid), 12 iterations, default SKFlow, against the fp32 oracle."""
    kw = dict(iters=12)
    sd = SO.synth_state_dict(SO.state_dict_shapes(), 1234)
    img = torch.from_numpy(synth.synth_images(1, 436, 1024, 4321, "smooth"))
    with torch.no_grad(), O.fp32_strict():
        ref = SO.raft_forward({k: v.to(DEV) for k, v in sd.items()}, img.to(DEV), **kw)["flows"].float().cpu()
    torch.cuda.empty_cache()
    model = _model(kw, sd, dtype)
    with torch.no_grad():
        out = model({"images": img.to(DEV, dtype)})
    d = (out["flows_fp32"].float().cpu() - ref).abs()
    _report(test="skflow_config_shape", dtype=str(dtype), err_flow=d.max().item(), mean_err=d.mean().item(), max_flow=ref.abs().max().item())
    assert d.max().item() < gate_max and d.mean().item() < gate_mean, f"max-abs {d.max().item():.4g} mean-abs {d.mean().item():.4g}"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_graph_replay_matches_eager(dtype):
    """The replayed graph computes what the eager forward does; they may differ by the run-to-run spread of the encoder's
    instance-norm statistics (atomic fp64 sums), far below the parity bounds."""
    recipe, _ = load_golden("e2e_skflow_heads2_pc_ragged")
    sd, img, kw = SO.e2e_inputs(recipe)
    model = _model(kw, sd, dtype)
    x = img.to(DEV, dtype)
    with torch.no_grad():
        model.use_cuda_graph = False
        eager = model({"images": x})["flows_fp32"].clone()
        model.use_cuda_graph = True
        model({"images": x})  # eager, counted
        model({"images": x})  # capture + replay
        replay = model({"images": x})["flows_fp32"]
    assert model.graph_replays >= 2
    d = (eager - replay).abs().max().item()
    _report(test="skflow_graph_vs_eager", dtype=str(dtype), err=d)
    assert d < (1e-3 if dtype == torch.float32 else 5e-2), d


def test_positional_grid_limit_raises_before_any_launch():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    sd = SO.synth_state_dict(SO.state_dict_shapes(), 3)
    model = _model(dict(iters=1, position_only=True), sd)
    img = torch.rand(1, 2, 3, 1288, 64, device=DEV)  # 161 x 8 grid
    torch.cuda.synchronize()
    before = lib.pfb_launch_count(-1)
    with pytest.raises(ValueError, match="160"):
        with torch.no_grad():
            model({"images": img})
    assert lib.pfb_launch_count(-1) == before
