"""GPU: SplatFlow against float64, the reference vectors and gma.

Kernel: pfb_softsplat_average against the float64 splat in fp32 / f16 / bf16, on the crafted flows of op_splatflow.npz and on a
strided 128-channel case like the model's.  End to end: the e2e_splatflow_* reference vectors in fp32, eagerly and replayed; a
two-frame splatflow holding a gma model's weights against that gma; three frames in f16 / bf16 at 436x1024 against the fp32 model.
"""
from argparse import Namespace

import numpy as np
import pytest
import torch

import splatflow_oracle as SO
from helpers import DEV, DTYPES, U, _model, _report, check_fp32_fixture, check_half_against_fp32, load_golden
from oracle import synth

pytestmark = pytest.mark.gpu


def _splat_check(x, flow, dtype, src_pad=0, dst_pad=0):
    """The kernel on x [B, C, H, W] (rounded to dtype) against the float64 splat of the rounded x.  Bound per element: the fp32
    arithmetic of the kernel (weights, products, the division; 1e-5 relative to the largest |x|) plus one rounding of the result to
    the storage type."""
    from ptlflow_b200 import ops

    b, c, h, w = x.shape
    xq = x.to(dtype).float()
    ref = SO.softsplat_average_f64(xq, flow)
    src = torch.zeros((b, h, w, c + 2 * src_pad), dtype=dtype, device=DEV)
    src[..., src_pad:src_pad + c] = xq.permute(0, 2, 3, 1).to(DEV, dtype)
    out = torch.full((b, h, w, c + 2 * dst_pad), 7.0, dtype=dtype, device=DEV)
    ops.softsplat_average(src, flow.to(DEV), out=out, channels=c, src_offset=src_pad, out_offset=dst_pad)
    torch.cuda.synchronize()
    got = out[..., dst_pad:dst_pad + c].float().cpu().permute(0, 3, 1, 2).double()
    bound = 1e-5 * max(1.0, xq.abs().max().item()) + U[dtype] * ref.abs()
    err = ((got - ref).abs() - bound).max().item()
    _report(test="softsplat_average", dtype=str(dtype), shape=list(x.shape), err=(got - ref).abs().max().item())
    assert err <= 0, err
    if dst_pad:
        assert (out[..., :dst_pad] == 7).all() and (out[..., dst_pad + c:] == 7).all()
    return got


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_splat_crafted_flows_vs_float64(dtype):
    x, flow = SO.op_splat_inputs()
    got = _splat_check(x, flow, dtype)
    assert (got == 0).all(dim=1).any()  # a pixel that receives nothing is 0, not NaN
    if dtype == torch.float32:  # the reference arithmetic: fp32 products summed in fp64
        np.testing.assert_allclose(got.float().numpy(), load_golden_splat(), atol=1e-6, rtol=0)


def load_golden_splat():
    from helpers import load_golden_arrays

    return load_golden_arrays("op_splatflow")["splat"]


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_splat_model_shape_vs_float64(dtype):
    """128 channels out of a 256-channel source into the upper half of a 256-channel destination, flows of a few px."""
    b, c, h, w = 2, 128, 11, 19
    x = torch.from_numpy(synth.synth_normal("gsplat/x", (b, c, h, w), 5))
    flow = torch.from_numpy(synth.synth_normal("gsplat/flow", (b, 2, h, w), 5, scale=3.0))
    _splat_check(x, flow, dtype, src_pad=64, dst_pad=128)


@pytest.mark.parametrize("name", SO.E2E)
def test_fp32_matches_reference_vectors(name):
    recipe, _ = load_golden(name)
    sd, img, kw = SO.e2e_inputs(recipe)
    check_fp32_fixture(_model("splatflow", sd, **kw), img, name, 1e-4)


def test_two_frames_equal_gma():
    """splatflow with two frames is GMA's forward (one head, content attention): the same weights under gma's names give gma's flow."""
    recipe, _ = load_golden("e2e_splatflow_three")
    sd, img, kw = SO.e2e_inputs(recipe)
    gsd = {k: v for k, v in SO._as_gma(sd, False).items() if not k.startswith("update.")}
    gma = _model("gma", {**gsd, **{k: v for k, v in _gma_pos(sd).items()}}, **kw)
    sf = _model("splatflow", sd, **kw)
    x = img[:, :2].contiguous().to(DEV)
    with torch.no_grad():
        a, b = gma({"images": x}), sf({"images": x})
    d = (a["flows"] - b["flows"]).abs().max().item()
    d_small = (a["flow_small"] - b["flow_small"]).abs().max().item()
    _report(test="splatflow_two_vs_gma", err=d, err_small=d_small)
    assert d < 1e-5 and d_small < 1e-5, (d, d_small)


def _gma_pos(sd):
    """gma's position tables (unused by its content attention, but part of its state dict)."""
    import gma_oracle as G

    shapes = {k: v for k, v in G.state_dict_shapes(1).items() if k.startswith("att.pos_emb")}
    return G.synth_state_dict(shapes, 0)


@pytest.mark.parametrize("frames", [2, 3])
def test_half_precision_at_436x1024(frames):
    """12 iterations per pair, random-init weights, f16 / bf16 against the fp32 model (max-abs / mean-abs px) with the gates of the
    other GMA-loop models (f16 8e-2 / 2e-2, bf16 5e-1 / 1e-1).  With three frames the bf16 max-abs gate is 1.5 px: pair (1, 2)
    refines from mf_t, the splat of pair (0, 1)'s bf16 motion features, so the two loops' rounding compounds; on this 28 px field the
    measured max-abs is 0.94 px at a mean-abs of 0.08 px (DESIGN.md section 5, SplatFlow)."""
    sd = SO.synth_state_dict(SO.state_dict_shapes(), 1234)
    img = torch.from_numpy(SO.images3(1, 436, 1024, 4321, "smooth", frames)).to(DEV)
    gates = {torch.float16: (8e-2, 2e-2), torch.bfloat16: (5e-1 if frames == 2 else 1.5, 1e-1)}
    check_half_against_fp32(lambda dtype: _model("splatflow", sd, dtype, iters=12), img, gates, f"splatflow {frames} frames 436x1024")
