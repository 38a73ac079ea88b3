"""GPU: SEA-RAFT against the oracle and the reference vectors.

Kernel: the fused depthwise convolution + LayerNorm against F.conv2d(groups=C) + F.layer_norm in fp32 / f16 / bf16, on grids
smaller than the kernel, from a strided channel slice and on inputs with a large common mean (the variance is taken about the
mean).  Update block: one iteration against sea_raft_oracle.iteration on the tensor path and with kernel_impl = 1.  End to end:
the e2e_sea_raft_* reference vectors in fp32 (eager and graph replay), the config-3 image size in half precision against the fp32
oracle, CUDA-graph replay against the eager forward, and the grid limit.
"""
import json
import os
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sea_raft_oracle as SR
from helpers import load_golden
from oracle import raft_oracle as O
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = os.environ.get("PFB_PARITY_REPORT")  # optional: one JSON line of measured errors per check
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


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


def _model(name, kwargs, sd, dtype=torch.float32, impl=0):
    import ptlflow_b200 as pb

    model = pb.get_model(name, args=Namespace(model=Namespace(**kwargs)))
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    model = model.eval().to(DEV)
    if dtype != torch.float32:
        model = model.to(dtype)
    model.kernel_impl = impl
    return model


# --------------------------------------------------------------------------------------
# depthwise convolution + LayerNorm
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("C,k", [(384, 7), (384, 3), (128, 7), (256, 1), (64, 31)])
def test_depthwise_layernorm_vs_torch(C, k, dtype):
    from ptlflow_b200 import ops

    w = _gen(f"dwln/w{k}", (C, 1, k, k), 1, scale=1.0 / k)
    b = _gen(f"dwln/b{k}", (C,), 2, scale=0.1)
    wt = w.reshape(C, k * k).t().contiguous().to(DEV)
    # 5x6: smaller than the 7x7 kernel; 17x23 reads a strided slice; 9x40 has a common mean of 300 on every channel
    for bsz, h, wd, pad, mean in ((2, 5, 6, 0, 0.0), (1, 17, 23, 8, 0.0), (2, 9, 40, 0, 300.0)):
        x = (_gen(f"dwln/x{h}", (bsz, C, h, wd), 3) + mean).to(dtype).float()
        y = F.conv2d(x, w, b, padding=k // 2, groups=C)
        ref = F.layer_norm(y.permute(0, 2, 3, 1), (C,), eps=1e-6)
        src = torch.zeros((bsz, h, wd, C + 2 * pad), dtype=dtype, device=DEV)
        src[..., pad:pad + C] = x.permute(0, 2, 3, 1).to(DEV, dtype)
        out = ops.depthwise_conv_layernorm(src, wt, b.to(DEV), k, channels=C, in_offset=pad)
        torch.cuda.synchronize()
        err = (out.float().cpu() - ref).abs().max().item()
        _report(test="dw_layernorm", k=k, C=C, dtype=str(dtype), grid=f"{h}x{wd}", mean=mean, err=err)
        # fp32 accumulation error, or about two roundings of the storage type (y, then the output) relative to the largest output
        tol = {torch.float32: 1e-4, torch.float16: 1e-3, torch.bfloat16: 8e-3}[dtype] * max(1.0, ref.abs().max().item())
        assert err < tol, (h, wd, mean, err)


def test_depthwise_layernorm_into_a_strided_output():
    from ptlflow_b200 import ops

    C, k = 384, 7
    w, b = _gen("dwln/w7s", (C, 1, k, k), 1, scale=1.0 / k), _gen("dwln/b7s", (C,), 2, scale=0.1)
    x = _gen("dwln/x7s", (1, C, 12, 20), 3)
    ref = F.layer_norm(F.conv2d(x, w, b, padding=3, groups=C).permute(0, 2, 3, 1), (C,), eps=1e-6)
    out = torch.full((1, 12, 20, C + 32), 7.0, device=DEV)
    ops.depthwise_conv_layernorm(x.permute(0, 2, 3, 1).contiguous().to(DEV), w.reshape(C, -1).t().contiguous().to(DEV), b.to(DEV), k,
                                 out=out, out_offset=16)
    torch.cuda.synchronize()
    assert (out[..., 16:16 + C].cpu() - ref).abs().max().item() < 1e-4
    assert (out[..., :16] == 7).all() and (out[..., 16 + C:] == 7).all()


# --------------------------------------------------------------------------------------
# one update iteration
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,h,w", SR.OP_GRIDS)
@pytest.mark.parametrize("dtype,impl", [(torch.float32, 0), (torch.float16, 0), (torch.bfloat16, 0), (torch.float16, 1)])
def test_update_iteration_vs_oracle(dtype, impl, b, h, w):
    """One SEA-RAFT update iteration (motion encoder, two ConvNeXt blocks, flow head, mask head) against sea_raft_oracle.iteration
    on the same storage-rounded inputs."""
    import ptlflow_b200 as pb
    from ptlflow_b200 import ops
    from ptlflow_b200.engine import SEARaftEngine

    sd, net, inp, corr, flow = SR.op_inputs(b, h, w)
    q = lambda t: t.to(dtype).float()  # noqa: E731
    net, inp, corr, flow = q(net), q(inp), q(corr), q(flow)
    n_ref, d_ref, m_ref = SR.iteration(net, inp, corr, flow, {k: v.float() for k, v in sd.items()})
    model = pb.get_model("sea_raft", args=Namespace(model=Namespace(iters=1)))
    model.load_state_dict(sd)
    model = model.to(DEV, dtype)
    eng = SEARaftEngine(model, 4, 128, 128, 4, 4, dtype, torch.device(DEV), impl=impl)
    coords0 = O.coords_grid(b, h, w)
    coords = ops.coords_to_pixel_major(coords0 + flow).to(DEV)
    net_d = net.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)
    corr_d = corr.permute(0, 2, 3, 1).contiguous().to(DEV, dtype)
    with torch.no_grad():
        mask = eng.update_iter(net_d, inp.permute(0, 2, 3, 1).contiguous().to(DEV, dtype), coords, corr=corr_d, want_mask=True)
    torch.cuda.synchronize()
    e_net = (net_d.float().cpu().permute(0, 3, 1, 2) - n_ref).abs().max().item()
    e_delta = ((coords.cpu().permute(0, 3, 1, 2) - coords0 - flow) - d_ref).abs().max().item()
    e_mask = (mask.float().cpu().permute(0, 3, 1, 2) - m_ref).abs().max().item()
    _report(test="sea_raft_update_iter", case=f"{h}x{w}", dtype=str(dtype), impl=impl, err_net=e_net, err_delta=e_delta, err_mask=e_mask,
            scale_net=n_ref.abs().max().item())
    # about 4x what one H100 measured (DESIGN.md section 5): fp32 1.5e-6 on every output; f16 7.5e-4 / 1.6e-4 / 7.1e-5 and bf16
    # 6.5e-3 / 1.2e-3 / 6.1e-4 on net / delta / mask (|net| <= 1.82)
    tol = {torch.float32: (1e-5, 1e-5, 1e-5), torch.float16: (3e-3, 6e-4, 3e-4), torch.bfloat16: (2.5e-2, 5e-3, 2.5e-3)}[dtype]
    assert e_net < tol[0] and e_delta < tol[1] and e_mask < tol[2], (e_net, e_delta, e_mask)


# --------------------------------------------------------------------------------------
# end to end
# --------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SR.E2E)
def test_fp32_matches_reference_vectors(name):
    recipe, g = load_golden(name)
    sd, img, mname, kw = SR.e2e_inputs(recipe)
    model = _model(mname, kw, sd)
    with torch.no_grad():
        out = model({"images": img.to(DEV)})
        out2 = model({"images": img.to(DEV)})  # captures, then replays the CUDA graph
        out3 = model({"images": img.to(DEV)})
    assert model.graph_replays >= 1
    err = np.abs(out["flows"].cpu().numpy() - g["flows"]).max()
    err_replay = max(np.abs(o["flows"].cpu().numpy() - g["flows"]).max() for o in (out2, out3))
    err_small = np.abs(out["flow_small"].cpu().numpy() - g["flow_small"]).max()
    _report(test="sea_raft_fp32_golden", case=name, err_flow=float(err), err_replay=float(err_replay), err_flow_small=float(err_small))
    assert out["flows"].shape == g["flows"].shape
    assert err < 1e-3 and err_replay < 1e-3 and err_small < 1e-3, f"{name}: max-abs flow error {err} / replay {err_replay} / small {err_small}"


def test_called_without_no_grad_and_training_guard():
    """The model is called as users call it, without torch.no_grad(), with iters = 0 (no update block) and with the default
    loop; training mode still raises NotImplementedError."""
    for name in ("e2e_sea_raft_iters0", "e2e_sea_raft_default_ragged"):
        recipe, g = load_golden(name)
        sd, img, mname, kw = SR.e2e_inputs(recipe)
        model = _model(mname, kw, sd)
        assert torch.is_grad_enabled()
        out = model({"images": img.to(DEV)})
        assert np.abs(out["flows"].detach().cpu().numpy() - g["flows"]).max() < 1e-3, name
        model.train()
        with pytest.raises(NotImplementedError):
            model({"images": img.to(DEV)})


def test_encoder_schedule_knobs():
    """enable_fp32_context() and encoder_chunk act on SEA-RAFT's encoders as on RAFT's."""
    recipe, g = load_golden("e2e_sea_raft_default_ragged")
    sd, img, mname, kw = SR.e2e_inputs(recipe)
    base = _model(mname, kw, sd, torch.float16)
    model = _model(mname, kw, sd)
    model.enable_fp32_context()
    model = model.half()
    model.encoder_chunk = 1
    assert model.__dict__.get("_cnet_fp32") is not None
    with torch.no_grad():
        d16 = np.abs(base({"images": img.to(DEV).half()})["flows_fp32"].cpu().numpy() - g["flows"]).max()
        out = model({"images": img.to(DEV).half()})
    d = np.abs(out["flows_fp32"].cpu().numpy() - g["flows"]).max()
    _report(test="sea_raft_fp32_context", err_flow=float(d), err_flow_f16=float(d16))
    assert d < d16 and d < 1e-2, (d, d16)


def test_half_model_returns_flows_and_flow_small():
    recipe, g = load_golden("e2e_sea_raft_default_ragged")
    sd, img, mname, kw = SR.e2e_inputs(recipe)
    model = _model(mname, kw, sd, torch.float16)
    with torch.no_grad():
        out = model({"images": img.to(DEV).half()})
    assert out["flows"].shape == g["flows"].shape and out["flows"].dtype == torch.float16
    assert out["flow_small"].shape == g["flow_small"].shape
    d = np.abs(out["flows_fp32"].cpu().numpy() - g["flows"])
    _report(test="sea_raft_f16_vs_fp32_ref", err_flow=float(d.max()), mean_err=float(d.mean()))
    assert d.max() < 0.1, d.max()


# Gates about 2-4x above what one H100 80GB HBM3 (400 W) measured, max-abs / mean-abs px (DESIGN.md section 5):
#   sea_raft (4 iterations, |flow| <= 5 px):   bf16 0.012 / 0.0031, f16 0.0017 / 0.0005
#   sea_raft_l (12 iterations, |flow| <= 90):  bf16 0.47 / 0.107,   f16 0.050 / 0.0091
@pytest.mark.parametrize("name,dtype,gate_max,gate_mean", [("sea_raft", torch.bfloat16, 5e-2, 1.2e-2), ("sea_raft", torch.float16, 8e-3, 2e-3),
                                                           ("sea_raft_l", torch.bfloat16, 1.0, 0.25), ("sea_raft_l", torch.float16, 0.15, 0.03)])
def test_config3_size_against_fp32_oracle(name, dtype, gate_max, gate_mean):
    """Config-3 image size (436x1024 -> 55x128 grid) against the fp32 oracle."""
    pretrain, iters = SR.PRETRAIN[name], (12 if name == "sea_raft_l" else 4)
    sd = SR.synth_state_dict(SR.state_dict_shapes(pretrain, iters), 1234)
    img = torch.from_numpy(synth.synth_images(1, 436, 1024, 4321, "smooth"))
    with torch.no_grad(), O.fp32_strict():
        ref = SR.forward({k: v.to(DEV) for k, v in sd.items()}, img.to(DEV), pretrain, iters)["flows"].float().cpu()
    torch.cuda.empty_cache()
    model = _model(name, {}, sd, dtype)
    with torch.no_grad():
        out = model({"images": img.to(DEV, dtype)})
    d = (out["flows_fp32"].float().cpu() - ref).abs()
    _report(test="sea_raft_config_shape", model=name, dtype=str(dtype), err_flow=d.max().item(), mean_err=d.mean().item(),
            max_flow=ref.abs().max().item())
    assert d.max().item() < gate_max and d.mean().item() < gate_mean, f"max-abs {d.max().item():.4g} mean-abs {d.mean().item():.4g}"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("name", ["e2e_sea_raft_default_ragged", "e2e_sea_raft_iters0"])
def test_graph_replay_matches_eager(name, dtype):
    recipe, _ = load_golden(name)
    sd, img, mname, kw = SR.e2e_inputs(recipe)
    model = _model(mname, kw, sd, dtype)
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
    _report(test="sea_raft_graph_vs_eager", case=name, dtype=str(dtype), err=d)
    assert d < (1e-4 if dtype == torch.float32 else 5e-2), d


def test_grid_limit_raises_before_any_launch():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    sd = SR.synth_state_dict(SR.state_dict_shapes(), 3)
    model = _model("sea_raft", {}, sd)
    img = torch.rand(1, 2, 3, 64, 96, device=DEV)  # 8 x 12 grid < 2**4
    torch.cuda.synchronize()
    before = lib.pfb_launch_count(-1)
    with pytest.raises(ValueError, match="2\\*\\*corr_levels"):
        with torch.no_grad():
            model({"images": img})
    assert lib.pfb_launch_count(-1) == before
