"""GPU: GMA's position-only, position-and-content and multi-head attention against the oracle and the reference vectors.

Operator level: the attention of every mode x heads on an N % 8 != 0 and an N % 8 == 0 grid, in fp32 and f16, on the tensor
path and with kernel_impl = 1; one update-block iteration with several heads (the per-head aggregate and the projection).
End to end: the e2e_gma_* reference vectors in fp32, and f16 / bf16 against them at the bounds test_gpu_e2e.py uses; the
config-3 image size in bf16 / f16 against the fp32 oracle at the bounds test_gpu_configs.py uses for cfg3_gma.
"""
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

import gma_oracle as GO
from helpers import load_golden
from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = os.environ.get("PFB_PARITY_REPORT")  # optional: one JSON line of measured errors per check
MODES = GO.MODES


def _report(**kw):
    if not REPORT:
        return
    try:
        os.makedirs(os.path.dirname(REPORT), exist_ok=True)
        with open(REPORT, "a") as f:
            f.write(json.dumps(kw) + "\n")
    except OSError:
        pass


def _model(kwargs, sd, dtype=torch.float32, impl=0):
    import ptlflow_b200 as pb

    model = pb.get_model("gma", args=Namespace(model=Namespace(**kwargs)))
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    model = model.eval().to(DEV)
    if dtype != torch.float32:
        model = model.to(dtype)
    model.kernel_impl = impl
    return model


def _engine(model, dtype, impl):
    from ptlflow_b200.engine import RaftEngine

    return RaftEngine(model.update_block, 2, 128, 128, 4, 4, dtype, torch.device(DEV), impl=impl, attention_module=model.att)


def _block_inputs(heads, seed):
    sd = GO.synth_state_dict({k: v for k, v in GO.state_dict_shapes(heads).items() if k.split(".")[0] in ("update_block", "att")}, seed)
    return sd


def _load_blocks(model, sd):
    model.update_block.load_state_dict({k[len("update_block."):]: v for k, v in sd.items() if k.startswith("update_block.")})
    model.att.load_state_dict({k[len("att."):]: v for k, v in sd.items() if k.startswith("att.")}, strict=False)


def _nhwc(x, dtype):
    return x.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)


ATT_CASES = [(mode, heads, dtype, impl) for mode in MODES for heads in (1, 2, 4)
             for dtype, impl in ((torch.float32, 0), (torch.float16, 0), (torch.float16, 1))]


@pytest.mark.parametrize("h,w", [(6, 9), (8, 16)])  # N = 54 (scalar rows, SIMT aggregate) and N = 128 (16-byte rows, tensor path)
@pytest.mark.parametrize("mode,heads,dtype,impl", ATT_CASES, ids=[f"{m}-h{k}-{str(d)[6:]}-impl{i}" for m, k, d, i in ATT_CASES])
def test_attention_vs_oracle(mode, heads, dtype, impl, h, w):
    import ptlflow_b200 as pb

    b = 2
    sd = _block_inputs(heads, 5)
    model = pb.get_model("gma", args=Namespace(model=Namespace(num_heads=heads, **MODES[mode])))
    _load_blocks(model, sd)
    model.update_block.to(DEV), model.att.to(DEV)
    model.kernel_impl = impl
    eng = _engine(model, dtype, impl)
    inp = torch.relu(torch.from_numpy(synth.synth_normal("gma/inp", (b, 128, h, w), 6)))
    ref = GO.attention(inp.to(dtype).float(), {k: v.to(dtype).float() for k, v in sd.items()}, heads, **MODES[mode])
    ref = ref.reshape(b, heads, h * w, h * w).transpose(0, 1)  # head-major like the device layout
    with torch.no_grad():
        attn = model._attention(_nhwc(inp, dtype), eng)
    assert attn.shape == (heads * b * h * w, h * w) and attn.dtype == dtype
    err = (attn.float().cpu().view(heads, b, h * w, h * w) - ref).abs().max().item()
    _report(test="gma_attention", case=f"{mode}_h{heads}_{h}x{w}", dtype=str(dtype), impl=impl, err=err)
    assert err < (2e-5 if dtype == torch.float32 else 2e-2)
    assert (attn.float().sum(-1) - 1).abs().max().item() < (1e-5 if dtype == torch.float32 else 5e-3)


@pytest.mark.parametrize("heads", [2, 4])
@pytest.mark.parametrize("h,w", [(9, 13), (8, 16)])  # N = 117 (SIMT aggregate in f16) and N = 128 (tensor path); 4 pyramid levels
@pytest.mark.parametrize("dtype,impl", [(torch.float32, 0), (torch.float32, 1), (torch.float16, 0), (torch.float16, 1)])
def test_multihead_update_iteration_vs_oracle(heads, h, w, dtype, impl):
    """One GMA update block with heads > 1 (per-head attn @ v into the concatenation, project + gamma AXPY, then the GRU and
    the heads) against gma_oracle.update_block on the same storage-rounded inputs."""
    import ptlflow_b200 as pb
    from ptlflow_b200 import ops

    b, planes = 2, 4 * 81
    sd = _block_inputs(heads, 8)
    model = pb.get_model("gma", args=Namespace(model=Namespace(num_heads=heads, position_and_content=True)))
    _load_blocks(model, sd)
    model.update_block.to(DEV), model.att.to(DEV)
    eng = _engine(model, dtype, impl)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, 9, scale=scale)).to(dtype).float()  # noqa: E731
    net, inp = torch.tanh(r("mh/net", (b, 128, h, w))), torch.relu(r("mh/inp", (b, 128, h, w)))
    corr, flow = r("mh/corr", (b, planes, h, w)), r("mh/flow", (b, 2, h, w), 3.0)
    sdq = {k: v.to(dtype).float() for k, v in sd.items()}
    attn = GO.attention(inp, sdq, heads, position_and_content=True)  # [b, heads, N, N]
    n_ref, _, d_ref = GO.update_block(net, inp, corr, flow, attn, sdq)
    coords0 = O.coords_grid(b, h, w)
    coords = ops.coords_to_pixel_major(coords0 + flow).to(DEV)
    net_d = _nhwc(net, dtype)
    attn_d = attn.transpose(0, 1).reshape(heads * b * h * w, h * w).to(DEV, dtype).contiguous()
    with torch.no_grad():
        eng.update_iter(net_d, _nhwc(inp, dtype), coords, corr=_nhwc(corr, dtype), attention=attn_d)
    torch.cuda.synchronize()
    e_net = (net_d.float().cpu().permute(0, 3, 1, 2) - n_ref).abs().max().item()
    e_delta = ((coords.cpu().permute(0, 3, 1, 2) - coords0 - flow) - d_ref).abs().max().item()
    _report(test="gma_multihead_update", case=f"h{heads}_{h}x{w}", dtype=str(dtype), impl=impl, err_net=e_net, err_delta=e_delta)
    # measured at 8x16: fp32 7e-7 (net) / 2e-6 (delta), f16 6e-4 / 1e-4
    tol = 1e-4 if dtype == torch.float32 else 5e-3
    assert e_net < tol and e_delta < tol


@pytest.mark.parametrize("name", GO.E2E)
def test_fp32_matches_reference_vectors(name):
    recipe, g = load_golden(name)
    sd, img, kw = GO.e2e_inputs(recipe)
    model = _model(kw, sd)
    with torch.no_grad():
        out = model({"images": img.to(DEV)})
        out2 = model({"images": img.to(DEV)})  # the second call replays the captured CUDA graph
    err = np.abs(out["flows"].cpu().numpy() - g["flows"]).max()
    err2 = np.abs(out2["flows"].cpu().numpy() - g["flows"]).max()
    err_small = np.abs(out["flow_small"].cpu().numpy() - g["flow_small"]).max()
    _report(test="fp32_golden", case=name, err_flow=float(err), err_replay=float(err2), err_flow_small=float(err_small))
    assert out["flows"].shape == g["flows"].shape
    assert err < 1e-3 and err2 < 1e-3 and err_small < 1e-3, f"{name}: max-abs flow error {err} / replay {err2} / small {err_small}"


@pytest.mark.parametrize("name", GO.E2E)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_against_fp32_reference(name, dtype):
    recipe, g = load_golden(name)
    sd, img, kw = GO.e2e_inputs(recipe)
    model = _model(kw, sd, dtype)
    with torch.no_grad():
        out = model({"images": img.to(DEV, dtype)})
    d = np.abs(out["flows_fp32"].cpu().numpy() - g["flows"])
    _report(test="half_vs_fp32_ref", case=name, dtype=str(dtype), err_flow=float(d.max()), mean_err=float(d.mean()))
    bound, mean_bound = (4e-2, 1e-2) if dtype == torch.float16 else (3e-1, 6e-2)
    assert d.max() < bound and d.mean() < mean_bound, f"{name} {dtype}: max-abs {d.max()} mean-abs {d.mean()}"


@pytest.mark.parametrize("dtype,gate_max,gate_mean", [(torch.bfloat16, 5e-1, 1e-1), (torch.float16, 8e-2, 2.5e-2)])
def test_config3_size_position_and_content_heads2(dtype, gate_max, gate_mean):
    """BASELINE config 3 image size (436x1024 -> 55x128 grid), position_and_content with two heads, against the fp32 oracle."""
    kw = dict(iters=12, num_heads=2, position_and_content=True)
    sd = GO.synth_state_dict(GO.state_dict_shapes(2), 1234)
    img = torch.from_numpy(synth.synth_images(1, 436, 1024, 4321, "smooth"))
    with torch.no_grad(), O.fp32_strict():
        ref = GO.raft_forward({k: v.to(DEV) for k, v in sd.items()}, img.to(DEV), **kw)["flows"].float().cpu()
    torch.cuda.empty_cache()
    model = _model(kw, sd, dtype)
    with torch.no_grad():
        out = model({"images": img.to(DEV, dtype)})
        out2 = model({"images": img.to(DEV, dtype)})
    d = (out["flows_fp32"].float().cpu() - ref).abs()
    d2 = (out2["flows_fp32"].float().cpu() - ref).abs()
    _report(test="config_shape", case="cfg3_gma_pc_h2", dtype=str(dtype), err_flow=d.max().item(), mean_err=d.mean().item(),
            err_replay=d2.max().item(), max_flow=ref.abs().max().item())
    assert d.max().item() < gate_max and d.mean().item() < gate_mean, f"max-abs {d.max().item():.4g} mean-abs {d.mean().item():.4g}"
    assert d2.max().item() < gate_max


@pytest.mark.parametrize("flags", [{"position_only": True}, {"position_and_content": True, "num_heads": 2}])
def test_positional_grid_limit_raises_before_any_launch(flags):
    from ptlflow_b200 import _lib

    lib = _lib.load()
    sd = GO.synth_state_dict(GO.state_dict_shapes(flags.get("num_heads", 1)), 3)
    model = _model(dict(iters=1, **flags), sd)
    img = torch.rand(1, 2, 3, 1288, 64, device=DEV)  # 161 x 8 grid
    torch.cuda.synchronize()
    before = lib.pfb_launch_count(-1)
    with pytest.raises(ValueError, match="160"):
        with torch.no_grad():
            model({"images": img})
    assert lib.pfb_launch_count(-1) == before
    content = _model(dict(iters=1), synth.synth_state_dict(O.state_dict_shapes("gma"), 3))
    with torch.no_grad():
        out = content({"images": img})
    assert out["flows"].shape == (1, 1, 2, 1288, 64) and torch.isfinite(out["flows"]).all()
