"""Flow1D on top of oracle/raft_oracle.py (TEST INFRASTRUCTURE, like oracle/): the sine position embedding, the 1D attention, the row /
column volumes and their 1D lookup written from their definitions, the forward, and the recipes of the fixtures
tests/make_flow1d_golden.py writes.

Written from the formulas of ptlflow/models/flow1d/{position,attention,correlation,flow1d}.py, fp32 on the CPU:
  pos:        channels 0..C/2-1 from the row index, C/2..C-1 from the column index; e = (i+1)/(n+1e-6) 2 pi, channel j of a half is
              sin(e / d_j) (j even) or cos(e / d_j) (j odd), d_j = 10000^(2 floor(j/2) / (C/2))
  attention:  q = Wq (f1 + pos) + bq, k = Wk (f2 + pos) + bk, v = f2;  out = softmax_l(q . k_l / sqrt(C)) v_l along the row
              (y_attention False) or the column;  double_cross_attn: f1 first goes through self_attn (the other axis, v = f1)
  volumes:    corr_x[b,y,x,x'] = f1[b,y,x] . feature2_y[b,y,x'] / sqrt(C);  corr_y[b,y,x,y'] = f1[b,y,x] . feature2_x[b,y',x] / sqrt(C)
  lookup:     sample p = c + d, d = -r..r, of a query's row: (1 - a) v[x0] + a v[x0 + 1], x0 = floor(p), taps outside the row are 0
  loop:       RAFT's BasicUpdateBlock over [corr_x taps | corr_y taps], convex 8x upsample of the last iteration
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]

# end-to-end fixtures: (name, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_flow1d_default", dict(iters=4), 1, 64, 96, "smooth", 211, 221, False),
    ("e2e_flow1d_ragged", dict(iters=3), 1, 61, 93, "smooth", 212, 222, False),
    ("e2e_flow1d_r8", dict(corr_radius=8, iters=3), 1, 64, 128, "smooth", 213, 223, False),
    ("e2e_flow1d_short", dict(iters=2), 1, 64, 384, "smooth", 214, 224, False),
    ("e2e_flow1d_warm", dict(iters=3), 1, 64, 96, "smooth", 215, 225, True),
    ("e2e_flow1d_b2", dict(iters=2), 2, 48, 80, "noise", 216, 226, False),
]
E2E = [c[0] for c in E2E_CASES]
OP_SEED = 231
OP_RADIUS = 4


def recipe_of(case) -> dict:
    name, kw, b, h, w, kind, ws, iseed, warm = case
    return dict(model="flow1d", kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm)


def state_dict_shapes(radius: int = 32):
    """The reference's state_dict names and shapes (written by tests/make_flow1d_golden.py for the default radius 32)."""
    import json
    import os

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "state_shapes_flow1d.json")) as f:
        shapes = {k: tuple(v) for k, v in json.load(f).items()}
    shapes["update_block.encoder.convc1.weight"] = (256, 2 * (2 * radius + 1), 1, 1)
    return shapes


def synth_state_dict(radius: int, seed: int) -> SD:
    return synth.synth_state_dict(state_dict_shapes(radius), seed)


# --------------------------------------------------------------------------------------
# operators
# --------------------------------------------------------------------------------------
def position(H: int, W: int, C: int) -> Tensor:
    """[C, H, W] fp32."""
    npf = C // 2
    d = 10000.0 ** (2.0 * (torch.arange(npf, dtype=torch.float64) // 2) / npf)

    def half(n: int) -> Tensor:  # [npf, n]
        e = torch.arange(1, n + 1, dtype=torch.float64) / (n + 1e-6) * (2 * math.pi)
        a = e[None, :] / d[:, None]
        even = (torch.arange(npf) % 2 == 0)[:, None]
        return torch.where(even, torch.sin(a), torch.cos(a))

    py, px = half(H)[:, :, None].expand(npf, H, W), half(W)[:, None, :].expand(npf, H, W)
    return torch.cat([py, px], 0).float()


def _conv1x1(x: Tensor, sd: SD, name: str) -> Tensor:
    return F.conv2d(x, sd[name + ".weight"], sd[name + ".bias"])


def attention1d(sd: SD, p: str, f1: Tensor, f2: Tensor, pos: Tensor, y_attention: bool, double: bool) -> Tensor:
    """Attention1D (p = "attn_x." etc.) on NCHW maps -> [B, C, H, W]."""
    if double:
        f1 = attention1d(sd, p + "self_attn.", f1, f1, pos, not y_attention, False)
    q, k, v = _conv1x1(f1 + pos, sd, p + "query_conv"), _conv1x1(f2 + pos, sd, p + "key_conv"), f2
    s = 1.0 / math.sqrt(f1.shape[1])
    if y_attention:  # along the column: key index z runs over y
        a = torch.softmax(torch.einsum("bcyx,bczx->bxyz", q, k) * s, dim=-1)
        return torch.einsum("bxyz,bczx->bcyx", a, v)
    a = torch.softmax(torch.einsum("bcyx,bcyz->byxz", q, k) * s, dim=-1)
    return torch.einsum("byxz,bcyz->bcyx", a, v)


def volumes(f1: Tensor, f2_x: Tensor, f2_y: Tensor):
    """(corr_x [B*H*W, W], corr_y [B*H*W, H])."""
    b, c, h, w = f1.shape
    s = 1.0 / math.sqrt(c)
    cx = torch.einsum("bcyx,bcyz->byxz", f1, f2_y) * s
    cy = torch.einsum("bcyx,bczx->byxz", f1, f2_x) * s
    return cx.reshape(b * h * w, w), cy.reshape(b * h * w, h)


def lookup_row(corr: Tensor, c: Tensor, radius: int) -> Tensor:
    """corr [N, L], c [N] -> [N, 2r+1]: an explicit 2-tap gather at c + d."""
    n, L = corr.shape
    p = c[:, None].double() + torch.arange(-radius, radius + 1, dtype=torch.float64)[None, :]
    x0 = torch.floor(p)
    a = (p - x0).to(corr.dtype)
    out = torch.zeros(n, 2 * radius + 1, dtype=corr.dtype)
    for off, wgt in ((0, 1 - a), (1, a)):
        xi = x0 + off
        ok = (xi >= 0) & (xi <= L - 1)
        idx = xi.clamp(0, L - 1).long()
        out = out + torch.gather(corr, 1, idx) * wgt * ok.to(corr.dtype)
    return out


def lookup(corr_x: Tensor, corr_y: Tensor, coords: Tensor, radius: int) -> Tensor:
    """coords [B, 2, H, W] -> [B, 2 (2r+1), H, W] = [corr_x taps | corr_y taps]."""
    b, _, h, w = coords.shape
    lx = lookup_row(corr_x, coords[:, 0].reshape(-1), radius)
    ly = lookup_row(corr_y, coords[:, 1].reshape(-1), radius)
    return torch.cat([lx, ly], 1).reshape(b, h, w, -1).permute(0, 3, 1, 2).contiguous()


def correlation(sd: SD, f1: Tensor, f2: Tensor):
    """(corr_x, corr_y, feature2_x, feature2_y) of flow1d.py:170-190."""
    pos = position(f1.shape[2], f1.shape[3], f1.shape[1])[None]
    f2_x = attention1d(sd, "attn_x.", f1, f2, pos, False, True)
    f2_y = attention1d(sd, "attn_y.", f1, f2, pos, True, True)
    cx, cy = volumes(f1, f2_x, f2_y)
    return cx, cy, f2_x, f2_y


def forward(sd: SD, images: Tensor, radius: int = 32, iters: int = 32, flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    x, pads = O.preprocess(images)
    b = x.shape[0]
    fm = O.encoder(torch.cat([x[:, 0], x[:, 1]], 0), sd, "fnet.", "instance", False)
    f1, f2 = fm[:b], fm[b:]
    cx, cy, _, _ = correlation(sd, f1, f2)
    cn = O.encoder(x[:, 0], sd, "cnet.", "batch", False)
    net, inp = torch.tanh(cn[:, :128]), torch.relu(cn[:, 128:])
    H, W = f1.shape[-2:]
    coords0 = O.coords_grid(b, H, W)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    mask = None
    for _ in range(iters):
        net, mask, delta = O.basic_update_block(net, inp, lookup(cx, cy, coords1, radius), coords1 - coords0, sd)
        coords1 = coords1 + delta
    flows = O.unpad(O.convex_upsample(coords1 - coords0, mask), pads)
    return {"flows": flows[:, None], "flow_small": coords1 - coords0}


def e2e_inputs(recipe):
    kw = dict(recipe["kwargs"])
    sd = synth_state_dict(kw.get("corr_radius", 32), recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


def forward_recipe(recipe, flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(sd, img, kw.get("corr_radius", 32), kw.get("iters", 32), flow_init)


def op_inputs():
    """Inputs of op_flow1d.npz (default-width weights, radius OP_RADIUS for the update block): features f1, f2 [2,256,6,9];
    coordinates with fractional, out-of-range and far-out-of-range entries; one update iteration's (net, inp, corr, flow)."""
    sd = synth_state_dict(OP_RADIUS, OP_SEED)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    K = 2 * OP_RADIUS + 1
    x = {
        "f1": r("f1dop/f1", (2, 256, 6, 9)),
        "f2": r("f1dop/f2", (2, 256, 6, 9)),
        "net": torch.tanh(r("f1dop/net", (2, 128, 6, 9))),
        "inp": torch.relu(r("f1dop/inp", (2, 128, 6, 9))),
        "corr": r("f1dop/corr", (2, 2 * K, 6, 9)),
        "flow": r("f1dop/flow", (2, 2, 6, 9), 3.0),
    }
    coords = O.coords_grid(2, 6, 9) + r("f1dop/coords", (2, 2, 6, 9), 4.0)
    coords[0, :, 0, :3] = torch.tensor([[-1e4, 3e4, 7.0], [2.5e4, -3e4, 2.0]])  # far out of range
    coords[1, :, 1, :4] = torch.tensor([[0.0, 8.0, -1.0, 9.0], [0.0, 5.0, -1.0, 6.0]])  # integers at and just past the edges
    x["coords"] = coords
    return sd, x


def np32(t: Tensor) -> np.ndarray:
    return t.detach().float().cpu().numpy().astype(np.float32)
