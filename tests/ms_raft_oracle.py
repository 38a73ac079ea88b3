"""MS-RAFT+ on top of the oracle (TEST INFRASTRUCTURE, like oracle/): group norm, the U-Net pyramid encoders, the four-scale loop with
its coordinate handover, downflow, the state-dict shapes and the recipes of the fixtures tests/make_ms_raft_golden.py writes.

Written from the formulas of ptlflow/models/ms_raft_plus/{extractor,update,ms_raft_plus}.py over oracle/raft_oracle.py, fp32 on
the CPU:
  block:     y = relu(GN(conv2(relu(GN(conv1 x)))));  x' = GN(down(x)) at stride 2;  out = y if the channels change at stride 1,
             else relu(x' + y)  (GN = GroupNorm(C / 8, C) with its affine; the conv bias stays, it is not removed by a group mean)
  encoder:   e1..e4 = layer1..4 after relu(GN(conv1 7x7/2)), e4 = conv2(layer4);  u2 = up2(cat[2x(e4), e3]), u1 = up1(cat[2x(u2), e2]),
             u0 = up0(cat[2x(u1), e1])  (2x = bilinear, align_corners=False)  ->  [e4, u2, u1, u0] at 1/16, 1/8, 1/4, 1/2
  scale i:   lookups of 2 levels from fmap1 / fmap2 of the scale, scaled by 1/sqrt(C);  RAFT's update block;  at the first iteration
             of scale i >= 1, coords = convex2x(coords, previous mask) (absolute coordinates, zero-padded taps)
  output:    flows = convex2x(coords - grid, last mask) un-padded;  flow_small = downflow(flows, 1/16)
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]

# end-to-end fixtures: (name, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_ms_raft_p_default", dict(), 1, 64, 96, "smooth", 71, 81, False),
    ("e2e_ms_raft_p_ragged_b2", dict(), 2, 100, 150, "smooth", 72, 82, False),
    ("e2e_ms_raft_p_volume", dict(alternate_corr=False), 1, 64, 96, "smooth", 73, 83, False),
    ("e2e_ms_raft_p_l3r3", dict(lookup_pyramid_levels=3, lookup_radius=3), 1, 128, 192, "smooth", 74, 84, False),
    ("e2e_ms_raft_p_iters1212", dict(iters=(1, 2, 1, 2)), 1, 64, 96, "noise", 75, 85, False),
    ("e2e_ms_raft_p_warm", dict(), 1, 64, 96, "smooth", 76, 86, True),
]
E2E = [c[0] for c in E2E_CASES]
OP_SEED = 93


def recipe_of(case) -> dict:
    name, kw, b, h, w, kind, ws, iseed, warm = case
    return dict(model="ms_raft_p", kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm)


# --------------------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------------------
def _conv(s, name: str, cout: int, cin: int, k: int) -> None:
    s[name + ".weight"], s[name + ".bias"] = (cout, cin, k, k), (cout,)


def _gn(s, name: str, c: int) -> None:
    s[name + ".weight"], s[name + ".bias"] = (c,), (c,)


def _encoder_shapes(s, p: str, out: int, up: Tuple[int, int, int]) -> None:
    _gn(s, p + "norm1", 64)
    _conv(s, p + "conv1", 64, 3, 7)

    def layer(name, cin, dim, stride):
        for i, (a, st) in enumerate(((cin, stride), (dim, 1))):
            q = f"{p}{name}.{i}."
            _conv(s, q + "conv1", dim, a, 3)
            _conv(s, q + "conv2", dim, dim, 3)
            _gn(s, q + "norm1", dim)
            _gn(s, q + "norm2", dim)
            if st != 1:  # norm3 and downsample.1 are one module under two names
                _gn(s, q + "norm3", dim)
                _conv(s, q + "downsample.0", dim, a, 1)
                _gn(s, q + "downsample.1", dim)

    layer("layer1", 64, 64, 1)
    layer("layer2", 64, 96, 2)
    layer("layer3", 96, 128, 2)
    layer("layer4", 128, 160, 2)
    _conv(s, p + "conv2", out, 160, 1)
    layer("up_layer2", out + 128, up[0], 1)
    layer("up_layer1", up[0] + 96, up[1], 1)
    layer("up_layer0", up[1] + 64, up[2], 1)


def state_dict_shapes(levels: int = 2, radius: int = 4) -> Dict[str, Tuple[int, ...]]:
    """The reference MS-RAFT+'s state_dict names and shapes (ms_raft_plus.py:103-109, extractor.py, update.py:119-140)."""
    s: Dict[str, Tuple[int, ...]] = {}
    _encoder_shapes(s, "fnet.", 256, (128, 96, 64))
    _encoder_shapes(s, "cnet.", 256, (256, 256, 256))
    e = "update_block.encoder."
    for name, cout, cin, k in (("convc1", 256, levels * (2 * radius + 1) ** 2, 1), ("convc2", 192, 256, 3), ("convf1", 128, 2, 7),
                               ("convf2", 64, 128, 3), ("conv", 126, 256, 3)):
        _conv(s, e + name, cout, cin, k)
    g = "update_block.gru."
    for i, (kh, kw) in (("1", (1, 5)), ("2", (5, 1))):
        for t in "zrq":
            s[f"{g}conv{t}{i}.weight"], s[f"{g}conv{t}{i}.bias"] = (128, 384, kh, kw), (128,)
    _conv(s, "update_block.flow_head.conv1", 256, 128, 3)
    _conv(s, "update_block.flow_head.conv2", 2, 256, 3)
    _conv(s, "update_block.mask.0", 256, 128, 3)
    _conv(s, "update_block.mask.2", 36, 256, 1)
    return s


def synth_state_dict(shapes, seed: int) -> SD:
    """oracle.synth weights: kaiming encoders (every stage is renormalised by its group norm), GroupNorm weight 1 + 0.1 N and bias
    0.05 N (not the identity), update block at torch's default-init variance."""
    return synth.synth_state_dict(shapes, seed)


def e2e_inputs(recipe):
    """(state_dict, images, kwargs) of an e2e_ms_raft_p_* fixture."""
    kw = dict(recipe["kwargs"])
    sd = synth_state_dict(state_dict_shapes(kw.get("lookup_pyramid_levels", 2), kw.get("lookup_radius", 4)), recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


def op_inputs():
    """Inputs of op_ms_raft_p.npz: state dict, a 1/4-scale feature map for the stride-2 block, the up-layer inputs, one update
    iteration's (net, inp, corr, flow) and a (coords, mask) pair for the convex 2x."""
    sd = synth_state_dict(state_dict_shapes(), OP_SEED)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    x = {
        "block_in": r("msop/block_in", (2, 64, 12, 20)),
        "up_coarse": r("msop/up_coarse", (2, 128, 5, 7)),
        "up_skip": r("msop/up_skip", (2, 96, 10, 14)),
        "net": r("msop/net", (2, 128, 6, 9)),
        "inp": r("msop/inp", (2, 128, 6, 9)),
        "corr": r("msop/corr", (2, 162, 6, 9)),
        "flow": r("msop/flow", (2, 2, 6, 9), 3.0),
        "mask": r("msop/mask", (2, 36, 6, 9), 2.0),
    }
    x["coords"] = O.coords_grid(2, 6, 9) + r("msop/coords", (2, 2, 6, 9), 4.0)
    return sd, x


# --------------------------------------------------------------------------------------
# blocks
# --------------------------------------------------------------------------------------
def group_norm(x: Tensor, sd: SD, name: str) -> Tensor:
    c = x.shape[1]
    return F.group_norm(x, c // 8, sd[name + ".weight"], sd[name + ".bias"], eps=1e-5)


def residual_block(x: Tensor, sd: SD, p: str, stride: int) -> Tensor:
    y = torch.relu(group_norm(O._conv(x, sd, p + "conv1", stride=stride, padding=1), sd, p + "norm1"))
    y = torch.relu(group_norm(O._conv(y, sd, p + "conv2", padding=1), sd, p + "norm2"))
    if stride != 1:
        x = group_norm(O._conv(x, sd, p + "downsample.0", stride=stride), sd, p + "downsample.1")
    if x.shape[1] != y.shape[1]:
        return y
    return torch.relu(x + y)


def layer(x: Tensor, sd: SD, p: str, stride: int) -> Tensor:
    return residual_block(residual_block(x, sd, p + ".0.", stride), sd, p + ".1.", 1)


def up2(x: Tensor) -> Tensor:
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False)


def up_layer(coarse: Tensor, skip: Tensor, sd: SD, p: str) -> Tensor:
    return layer(torch.cat([up2(coarse), skip], 1), sd, p, 1)


def pyramid_encoder(x: Tensor, sd: SD, p: str):
    x = torch.relu(group_norm(O._conv(x, sd, p + "conv1", stride=2, padding=3), sd, p + "norm1"))
    e1 = layer(x, sd, p + "layer1", 1)
    e2 = layer(e1, sd, p + "layer2", 2)
    e3 = layer(e2, sd, p + "layer3", 2)
    e4 = O._conv(layer(e3, sd, p + "layer4", 2), sd, p + "conv2")
    u2 = up_layer(e4, e3, sd, p + "up_layer2")
    u1 = up_layer(u2, e2, sd, p + "up_layer1")
    u0 = up_layer(u1, e1, sd, p + "up_layer0")
    return [e4, u2, u1, u0]


def convex_up2(v: Tensor, mask: Tensor) -> Tensor:
    """v [B,2,H,W] (flow or absolute coordinates), mask [B,36,H,W] (channel tap*4 + sy*2 + sx) -> [B,2,2H,2W]: softmax over the
    taps of the zero-padded 3x3 neighbourhood of 2 v."""
    b, _, h, w = v.shape
    m = torch.softmax(mask.view(b, 9, 2, 2, h, w), dim=1)
    f = F.pad(2.0 * v, (1, 1, 1, 1))
    out = torch.zeros(b, 2, 2, 2, h, w, dtype=v.dtype)
    for tap in range(9):
        dy, dx = tap // 3, tap % 3
        out = out + m[:, tap][:, None] * f[:, :, dy : dy + h, dx : dx + w][:, :, None, None]
    return out.permute(0, 1, 4, 2, 5, 3).reshape(b, 2, 2 * h, 2 * w)


def downflow(flow: Tensor, factor: float = 0.0625) -> Tensor:
    h, w = flow.shape[-2:]
    nh, nw = int(factor * h), int(factor * w)
    r = F.interpolate(flow, size=(nh, nw), mode="bilinear", align_corners=True)
    return torch.cat([r[:, :1] * (nw / w), r[:, 1:] * (nh / h)], 1)


def update_block(net, inp, corr, flow, sd: SD):
    """-> (net, mask [B,36,H,W] (x0.25), delta): RAFT's BasicUpdateBlock with the 2x mask head."""
    return O.basic_update_block(net, inp, corr, flow, sd)


def forward(sd: SD, images: Tensor, iters=(4, 6, 5, 10), levels: int = 2, radius: int = 4, alternate_corr: bool = True,
            flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    x = torch.flip((images + (-0.5)) * 2.0, dims=[-3])
    pads = O.pad_amounts(x.shape[-2], x.shape[-1], 16)
    b = x.shape[0]
    x = F.pad(x.reshape(2 * b, *x.shape[2:]), pads, mode="replicate").reshape(b, 2, 3, x.shape[-2] + pads[2] + pads[3], -1)
    fp = pyramid_encoder(torch.cat([x[:, 0], x[:, 1]], 0), sd, "fnet.")
    cp = pyramid_encoder(x[:, 0], sd, "cnet.")
    H, W = fp[0].shape[-2:]
    coords0 = O.coords_grid(b, H, W)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    mask = None
    for i in range(4):
        f1, f2 = fp[i][:b], fp[i][b:]
        if alternate_corr:
            lookup = lambda c: O.alt_corr_lookup(f1, f2, c, radius, levels)  # noqa: E731
        else:
            pyr = O.corr_pyramid(O.corr_volume(f1, f2), levels)
            lookup = lambda c: O.corr_lookup(pyr, c, radius)  # noqa: E731
        net, inp = torch.tanh(cp[i][:, :128]), torch.relu(cp[i][:, 128:])
        if i > 0:
            coords1 = convex_up2(coords1, mask)
            coords0 = O.coords_grid(b, *coords1.shape[-2:])
        for _ in range(iters[i]):
            net, mask, delta = update_block(net, inp, lookup(coords1), coords1 - coords0, sd)
            coords1 = coords1 + delta
    flows = O.unpad(convex_up2(coords1 - coords0, mask), pads)
    return {"flows": flows[:, None], "flow_small": downflow(flows)}


def forward_recipe(recipe, flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(sd, img, tuple(kw.get("iters", (4, 6, 5, 10))), kw.get("lookup_pyramid_levels", 2), kw.get("lookup_radius", 4),
                       kw.get("alternate_corr", True), flow_init)


def lookup_scale(c: int) -> float:
    return 1.0 / math.sqrt(c)


def np32(t: Tensor) -> np.ndarray:
    return t.detach().cpu().numpy().astype(np.float32)
