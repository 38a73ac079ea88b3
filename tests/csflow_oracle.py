"""CSFlow on top of oracle/raft_oracle.py (TEST INFRASTRUCTURE, like oracle/): the strip module, the 2-channel pyramid, its lookup, the
initial strip flow and the forward, written from their definitions, and the recipes of the fixtures tests/make_csflow_golden.py writes.

Written from the formulas of ptlflow/models/csflow/csflow.py, fp32 on the CPU:
  strips:   f1w, f1h, g2w, g2h = relu(bn(conv1x1(.))) of fmap1 / fmap2 (csflow.py:239-260); kw = column means of g2w, kh = row means of
            g2h; sw[q, x2] = <f1w[q], kw[x2]>, sh[q, y2] = <f1h[q], kh[y2]>, unscaled (csflow.py:262-272)
  pyramid:  the 2-channel volume [<f1, f2> / sqrt(C), sw[x2] + sh[y2]] materialised in 4D and 2x2-pooled 3 times (csflow.py:445-466),
            so the library's separable tables are checked against something that does not share their algebra
  lookup:   RAFT's window on both channels of each level; per level [81 taps of the 4D channel | 81 of the strip channel], levels
            concatenated (csflow.py:468-493)
  init:     corr_init = (sum_y2 softmax(sh, singleton axis) sh, sum_x2 softmax(sw, singleton axis) sw), kept literally
            (csflow.py:176-190), added to the start coordinates after the warm start
  loop:     RAFT's BasicUpdateBlock over that lookup, convex 8x upsample of the last iteration
"""
from __future__ import annotations

import json
import os
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]
LEVELS = 4

# end-to-end fixtures: (name, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_csflow_default", dict(iters=4), 1, 128, 160, "smooth", 311, 321, False),
    ("e2e_csflow_ragged", dict(iters=3), 2, 129, 131, "noise", 312, 322, False),  # padded, 1/8 grid 17 x 17: floor pooling 17 -> 8
    ("e2e_csflow_r3", dict(corr_radius=3, iters=3), 1, 128, 128, "smooth", 313, 323, False),
    ("e2e_csflow_r6", dict(corr_radius=6, iters=2), 1, 136, 128, "smooth", 314, 324, False),
    ("e2e_csflow_warm", dict(iters=3), 1, 128, 160, "smooth", 315, 325, True),
]
E2E = [c[0] for c in E2E_CASES]
OP_SEED = 331
OP_GRID = (16, 17)  # the strip operators' 1/8 grid (levels 16x17, 8x8, 4x4, 2x2)
OP_LOOKUP_RADIUS = 1
OP_ITER_GRID = (8, 8)  # the update iteration's grid (radius 4: 648 lookup planes; the loop needs 4 levels of at least one pixel)
# The strip block's BatchNorm weights and biases are scaled by this factor (its ReLU outputs, and so f1w, f1h, kw, kh, shrink by it).
# With oracle.synth's unscaled recipe sw and sh are tens and the initial flow is hundreds of cells, so every lookup after it samples
# outside the volume.  Scaled, tests/make_csflow_golden.py measured sw and sh in [0.006, 0.058] and the initial flow in [0.12, 0.83]
# cells (both components) across the e2e fixtures.
STRIP_BN_SCALE = 0.02


def recipe_of(case) -> dict:
    name, kw, b, h, w, kind, ws, iseed, warm = case
    return dict(model="csflow", kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm)


def state_dict_shapes(radius: int = 4):
    """The reference's state_dict names and shapes (written by tests/make_csflow_golden.py for the default radius 4)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "state_shapes_csflow.json")) as f:
        shapes = {k: tuple(v) for k, v in json.load(f).items()}
    shapes["update_block.encoder.convc1.weight"] = (256, 2 * LEVELS * (2 * radius + 1) ** 2, 1, 1)
    return shapes


def synth_state_dict(radius: int, seed: int) -> SD:
    sd = synth.synth_state_dict(state_dict_shapes(radius), seed)
    for k in sd:
        if k.startswith("strip_corr_block_v2.") and (k.endswith("bn.weight") or k.endswith("bn.bias")):
            sd[k] = sd[k] * STRIP_BN_SCALE
    return sd


# --------------------------------------------------------------------------------------
# operators
# --------------------------------------------------------------------------------------
def conv_bn_relu(x: Tensor, sd: SD, p: str) -> Tensor:
    y = F.conv2d(x, sd[p + "conv.weight"])
    y = F.batch_norm(y, sd[p + "bn.running_mean"], sd[p + "bn.running_var"], sd[p + "bn.weight"], sd[p + "bn.bias"], training=False, eps=1e-5)
    return torch.relu(y)


def strip_maps(sd: SD, f1: Tensor, f2: Tensor, p: str = "strip_corr_block_v2."):
    """(sw [B,H,W,W2], sh [B,H,W,H2]) of NCHW features."""
    f1w, f1h = conv_bn_relu(f1, sd, p + "conv1_1."), conv_bn_relu(f1, sd, p + "conv1_2.")
    kw = conv_bn_relu(f2, sd, p + "conv2_1.").mean(dim=2)  # [B, C, W]
    kh = conv_bn_relu(f2, sd, p + "conv2_2.").mean(dim=3)  # [B, C, H]
    return torch.einsum("bcyx,bcz->byxz", f1w, kw), torch.einsum("bcyx,bcz->byxz", f1h, kh)


def corr_init(sw: Tensor, sh: Tensor) -> Tensor:
    """csflow.py:177-190 as written: both softmax calls over a singleton axis -> [B, 2, H, W]."""
    w5, h5 = sw.unsqueeze(3), sh.unsqueeze(4)  # B H W 1 W2, B H W H2 1
    flow_v = torch.sum(torch.softmax(w5, dim=3).mul(w5), dim=4).squeeze(dim=3)
    flow_u = torch.sum(torch.softmax(h5, dim=4).mul(h5), dim=3).squeeze(dim=3)
    return torch.stack((flow_u, flow_v), dim=1)


def pyramid(f1: Tensor, f2: Tensor, sw: Tensor, sh: Tensor):
    """The 4 levels of the 2-channel volume [B*H*W, 2, h_l, w_l], the strip channel materialised."""
    b, c, h, w = f1.shape
    strip = (sw[:, :, :, None, :] + sh[:, :, :, :, None]).reshape(b * h * w, 1, h, w)
    return O.corr_pyramid(torch.cat([O.corr_volume(f1, f2), strip], 1), LEVELS)


def lookup(pyr, coords: Tensor, radius: int) -> Tensor:
    """coords [B,2,H,W] -> [B, 2 L (2r+1)^2, H, W] in the reference's order: per level [4D taps | strip taps]."""
    b, _, h, w = coords.shape
    n, k = b * h * w, 2 * radius + 1
    d = torch.arange(-radius, radius + 1, dtype=coords.dtype)
    outs = []
    for lvl, vol in enumerate(pyr):
        px = (coords[:, 0].reshape(n, 1, 1) / 2**lvl + d.view(1, k, 1)).expand(n, k, k).reshape(n, k * k)
        py = (coords[:, 1].reshape(n, 1, 1) / 2**lvl + d.view(1, 1, k)).expand(n, k, k).reshape(n, k * k)
        for ch in range(2):
            outs.append(O._bilinear_zero(vol[:, ch], px, py).view(b, h, w, k * k))
    return torch.cat(outs, dim=-1).permute(0, 3, 1, 2).contiguous()


def forward(sd: SD, images: Tensor, radius: int = 4, iters: int = 32, flow_init: Optional[Tensor] = None, trace: Optional[dict] = None):
    x, pads = O.preprocess(images)
    b = x.shape[0]
    fm = O.encoder(torch.cat([x[:, 0], x[:, 1]], 0), sd, "fnet.", "instance", False)
    f1, f2 = fm[:b], fm[b:]
    cn = O.encoder(x[:, 0], sd, "cnet.", "batch", False)
    net, inp = torch.tanh(cn[:, :128]), torch.relu(cn[:, 128:])
    sw, sh = strip_maps(sd, f1, f2)
    pyr = pyramid(f1, f2, sw, sh)
    H, W = f1.shape[-2:]
    coords0 = O.coords_grid(b, H, W)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    init = corr_init(sw, sh)
    coords1 = coords1 + init
    if trace is not None:
        trace.update(sw=sw, sh=sh, corr_init=init)
    mask = None
    for _ in range(iters):
        net, mask, delta = O.basic_update_block(net, inp, lookup(pyr, coords1, radius), coords1 - coords0, sd)
        coords1 = coords1 + delta
    flows = O.unpad(O.convex_upsample(coords1 - coords0, mask), pads)
    return {"flows": flows[:, None], "flow_small": coords1 - coords0}


def e2e_inputs(recipe):
    kw = dict(recipe["kwargs"])
    sd = synth_state_dict(kw.get("corr_radius", 4), recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


def forward_recipe(recipe, flow_init: Optional[Tensor] = None, trace: Optional[dict] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(sd, img, kw.get("corr_radius", 4), kw.get("iters", 32), flow_init, trace)


def op_inputs():
    """Inputs of op_csflow.npz (default radius 4 weights): features f1, f2 [1,256,16,17] and
    coordinates with fractional, out-of-range and far-out-of-range entries for the strip operators; one update iteration's (net, inp,
    corr, flow) on an 8x8 grid."""
    sd = synth_state_dict(4, OP_SEED)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    h, w = OP_GRID
    hi, wi = OP_ITER_GRID
    x = {
        "f1": r("csop/f1", (1, 256, h, w)),
        "f2": r("csop/f2", (1, 256, h, w)),
        "net": torch.tanh(r("csop/net", (1, 128, hi, wi))),
        "inp": torch.relu(r("csop/inp", (1, 128, hi, wi))),
        "corr": r("csop/corr", (1, 2 * LEVELS * 81, hi, wi)),
        "flow": r("csop/flow", (1, 2, hi, wi), 3.0),
    }
    coords = O.coords_grid(1, h, w) + r("csop/coords", (1, 2, h, w), 6.0)
    coords[0, :, 0, :4] = torch.tensor([[-1e4, 3e4, 7.0, 16.0], [2.5e4, -3e4, 2.0, 15.0]])  # far out of range, and the last pixel
    coords[0, :, 1, :4] = torch.tensor([[0.0, 16.0, -1.0, 17.0], [0.0, 15.0, -1.0, 16.0]])  # integers at and just past the edges
    x["coords"] = coords
    return sd, x


def op_outputs(sd: SD, x) -> Dict[str, Tensor]:
    """The oracle's counterpart of make_csflow_golden.reference_ops."""
    sw, sh = strip_maps(sd, x["f1"], x["f2"])
    pyr = pyramid(x["f1"], x["f2"], sw, sh)
    out = {"sw": sw, "sh": sh, "corr_init": corr_init(sw, sh), f"lookup_r{OP_LOOKUP_RADIUS}": lookup(pyr, x["coords"], OP_LOOKUP_RADIUS)}
    net, mask, delta = O.basic_update_block(x["net"], x["inp"], x["corr"], x["flow"], sd)
    out.update(net=net, mask=mask, delta=delta)
    return out


def np32(t: Tensor) -> np.ndarray:
    return t.detach().float().cpu().numpy().astype(np.float32)
