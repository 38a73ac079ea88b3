"""SplatFlow on top of the GMA oracle (TEST INFRASTRUCTURE, like oracle/): the "average" forward splat, the two-pass forward over
three frames, the state-dict shapes, the three-frame synthetic images and the recipes of the fixtures tests/make_splatflow_golden.py
writes.

Written from the formulas of ptlflow/models/splatflow/splatflow.py:86-154, update.py:82-123 and softsplat.py:10-60, 435-468 over
the building blocks of oracle/raft_oracle.py and tests/gma_oracle.py.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch

import gma_oracle as G
from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]

# end-to-end fixtures: (name, model kwargs, batch, H, W, image kind, frames, weight seed, image seed, prev_preds given)
# (1/8 grids of at least 16 px per side: the reference's bilinear_sampler divides by H - 1 of the coarsest level)
E2E_CASES = [
    ("e2e_splatflow_two", dict(iters=6), 1, 128, 192, "smooth", 2, 31, 41, False),
    ("e2e_splatflow_three", dict(iters=6), 1, 128, 192, "smooth", 3, 32, 42, False),
    ("e2e_splatflow_three_b2", dict(iters=4), 2, 128, 160, "smooth", 3, 33, 43, False),
    ("e2e_splatflow_three_ragged", dict(iters=5), 1, 132, 164, "noise", 3, 34, 44, False),  # 17 x 21 grid, N % 8 != 0
    ("e2e_splatflow_prev", dict(iters=4), 1, 128, 160, "smooth", 3, 35, 45, True),
    ("e2e_splatflow_r3", dict(iters=4, corr_radius=3, corr_levels=3), 1, 128, 160, "smooth", 3, 36, 46, False),
]
E2E = [c[0] for c in E2E_CASES]


def recipe_of(case) -> dict:
    name, kw, b, h, w, kind, frames, ws, iseed, prev = case
    return dict(variant="splatflow", kwargs=kw, batch=b, height=h, width=w, kind=kind, frames=frames, wseed=ws, iseed=iseed, prev=prev)


# operator fixture op_splatflow.npz
OP_SEED = 91
OP_SPLAT_GRID = (2, 7, 9, 12)  # (batch, H, W, channels)
OP_ITER_GRID = (1, 8, 12)  # (batch, H, W) of the gru_sp update


# --------------------------------------------------------------------------------------
# inputs and weights
# --------------------------------------------------------------------------------------
def images3(batch: int, height: int, width: int, seed: int, kind: str, frames: int) -> np.ndarray:
    """Frames [B, T, 3, H, W] float32 in [0, 1), BGR.  "noise": i.i.d. uniform.  "smooth": box-blurred coarse noise as in
    oracle.synth.synth_images, frame t moved by t (+4, -3) px."""
    g = np.random.Generator(np.random.Philox(key=[int(seed) & 0xFFFFFFFF, 0x5F1A7]))
    if kind == "noise":
        return g.random((batch, frames, 3, height, width), dtype=np.float32)
    if kind != "smooth":
        raise ValueError(kind)
    m = 4 * frames  # margin: the last frame moves 4 (T - 1) px left
    ch, cw = height // 8 + 2 + m // 8 + 1, width // 8 + 2 + m // 8 + 1
    img = np.repeat(np.repeat(g.random((batch, 3, ch, cw), dtype=np.float32), 8, axis=2), 8, axis=3)
    k = 9
    for _ in range(2):
        c = np.cumsum(np.pad(img, ((0, 0), (0, 0), (k, 0), (0, 0))), axis=2, dtype=np.float64)
        img = ((c[:, :, k:] - c[:, :, :-k]) / k).astype(np.float32)
        c = np.cumsum(np.pad(img, ((0, 0), (0, 0), (0, 0), (k, 0))), axis=3, dtype=np.float64)
        img = ((c[:, :, :, k:] - c[:, :, :, :-k]) / k).astype(np.float32)
    y0, x0 = 8, 8 + m
    out = np.stack([img[:, :, y0 + 3 * t: y0 + 3 * t + height, x0 - 4 * t: x0 - 4 * t + width] for t in range(frames)], axis=1)
    lo, hi = out.min(), out.max()
    return ((out - lo) / max(hi - lo, 1e-6) * 0.999).astype(np.float32)


def images(recipe: dict) -> Tensor:
    return torch.from_numpy(images3(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"], recipe["frames"]))


def prev_flow_small(recipe: dict) -> Tensor:
    """The prev_preds flow_small of a ``prev`` case: any flow, since the model must ignore it."""
    b, h, w = recipe["batch"], -(-recipe["height"] // 8), -(-recipe["width"] // 8)
    return torch.from_numpy(synth.synth_normal("splatflow/prev", (b, 2, h, w), recipe["iseed"], scale=3.0))


def state_dict_shapes() -> Dict[str, Tuple[int, ...]]:
    """The reference's names: GMA's encoders, ``att.to_qk`` (no position tables) and ``update.*`` = GMA's update block plus gru_sp
    (640 input channels with the hidden state), flow_head_sp and mask_sp (splatflow.py:45-49, update.py:82-107)."""
    s = {}
    for k, v in G.state_dict_shapes(1).items():
        if k.startswith("att.pos_emb"):
            continue
        if k.startswith("update_block."):
            k = "update." + k[len("update_block."):]
        s[k] = v
    for k, v in list(s.items()):
        for part, sp in (("update.gru.", "update.gru_sp."), ("update.flow_head.", "update.flow_head_sp."), ("update.mask.", "update.mask_sp.")):
            if k.startswith(part):
                if part == "update.gru." and k.endswith("weight"):
                    v = (v[0], v[1] + 128) + tuple(v[2:])
                s[sp + k[len(part):]] = v
    return s


def synth_state_dict(shapes, seed: int) -> SD:
    """oracle.synth weights (Aggregate.gamma 0.5 + 0.1 N(0, 1), so the aggregate is live)."""
    return synth.synth_state_dict(shapes, seed)


def e2e_inputs(recipe):
    """(state_dict, images, kwargs) of an e2e_splatflow_* fixture."""
    return synth_state_dict(state_dict_shapes(), recipe["wseed"]), images(recipe), dict(recipe["kwargs"])


# --------------------------------------------------------------------------------------
# the splat
# --------------------------------------------------------------------------------------
def softsplat_average(x: Tensor, flow: Tensor) -> Tensor:
    """The "average" splat of softsplat.py:10-60, 435-468 on the CPU, line for line: x [B, C, H, W] fp32 with a ones channel
    appended, targets (x + u, y + v) and the four corners' bilinear weights in fp32, each product value * weight in fp32, added in
    fp64 at the in-image corners (index_add_), then .float(), zero normalisers set to 1 and an fp32 division."""
    x, flow = x.float(), flow.float()
    b, c, h, w = x.shape
    inp = torch.cat([x, x.new_ones(b, 1, h, w)], 1)
    gy, gx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    fx = gx.float()[None] + flow[:, 0]
    fy = gy.float()[None] + flow[:, 1]
    nwx, nwy = torch.floor(fx).to(torch.int64), torch.floor(fy).to(torch.int64)
    nex, ney, swx, swy, sex, sey = nwx + 1, nwy, nwx, nwy + 1, nwx + 1, nwy + 1
    weights = ((sex.float() - fx) * (sey.float() - fy), (fx - swx.float()) * (swy.float() - fy),
               (nex.float() - fx) * (fy - ney.float()), (fx - nwx.float()) * (fy - nwy.float()))
    out = torch.zeros(b, c + 1, h * w, dtype=torch.float64)
    for (cx, cy), wt in zip(((nwx, nwy), (nex, ney), (swx, swy), (sex, sey)), weights):
        ok = (cx >= 0) & (cx < w) & (cy >= 0) & (cy < h)
        for n in range(b):
            m = ok[n].reshape(-1)
            idx = (cy[n] * w + cx[n]).reshape(-1)[m]
            val = (inp[n].reshape(c + 1, -1) * wt[n].reshape(1, -1))[:, m]  # fp32 products
            out[n].index_add_(1, idx, val.double())
    out = out.float().reshape(b, c + 1, h, w)
    norm = out[:, -1:].clone()
    norm[norm == 0.0] = 1.0
    return out[:, :-1] / norm


def softsplat_average_f64(x: Tensor, flow: Tensor) -> Tensor:
    """The same splat as a brute-force float64 loop over source pixels (weights, products and sums in float64): the yardstick of
    the stand-in above and of the kernel."""
    x, flow = x.double(), flow.double()
    b, c, h, w = x.shape
    acc = torch.zeros(b, c + 1, h, w, dtype=torch.float64)
    for n in range(b):
        for y in range(h):
            for xx in range(w):
                tx, ty = xx + flow[n, 0, y, xx].item(), y + flow[n, 1, y, xx].item()
                x0, y0 = int(np.floor(tx)), int(np.floor(ty))
                for cx, cy, wt in ((x0, y0, (x0 + 1 - tx) * (y0 + 1 - ty)), (x0 + 1, y0, (tx - x0) * (y0 + 1 - ty)),
                                   (x0, y0 + 1, (x0 + 1 - tx) * (ty - y0)), (x0 + 1, y0 + 1, (tx - x0) * (ty - y0))):
                    if 0 <= cx < w and 0 <= cy < h:
                        acc[n, :c, cy, cx] += x[n, :, y, xx] * wt
                        acc[n, c, cy, cx] += wt
    norm = acc[:, c:].clone()
    norm[norm == 0] = 1.0
    return acc[:, :c] / norm


def op_splat_inputs():
    """(x [B, C, H, W], flow [B, 2, H, W]) of op_splatflow.npz: fractional, integer, negative and out-of-image targets, collisions
    (many sources onto one pixel) and pixels that receive nothing."""
    b, h, w, c = OP_SPLAT_GRID
    x = torch.from_numpy(synth.synth_normal("splat/x", (b, c, h, w), OP_SEED))
    flow = torch.from_numpy(synth.synth_normal("splat/flow", (b, 2, h, w), OP_SEED, scale=2.0))
    flow[0, :, 0, :] = torch.round(flow[0, :, 0, :])  # integer targets
    flow[0, 0, 1, :] = -20.0  # out of the image to the left
    flow[0, 1, 2, :] = 30.5  # below the image
    flow[1, 0, :3, :3] = 4.0 - torch.arange(3.0)[None, :]  # a 3 x 3 block collapsing onto column 4 ...
    flow[1, 1, :3, :3] = 5.0 - torch.arange(3.0)[:, None]  # ... row 5: collisions
    flow[1, :, 3:, 5:] = torch.tensor([-0.25, -0.75])[:, None, None]  # negative fractional motion
    return x, flow


def op_iter_inputs():
    """(state dict, net, inp, corr, flow, attn, mf_t) of the gru_sp update in op_splatflow.npz."""
    b, h, w = OP_ITER_GRID
    sd = synth_state_dict({k: v for k, v in state_dict_shapes().items() if k.startswith(("update.", "att."))}, OP_SEED)
    g = lambda n, shp, s=1.0: torch.from_numpy(synth.synth_normal("splatit/" + n, shp, OP_SEED, scale=s))  # noqa: E731
    net = torch.tanh(g("net", (b, 128, h, w)))
    inp = torch.relu(g("inp", (b, 128, h, w)))
    corr = g("corr", (b, 324, h, w))
    flow = g("flow", (b, 2, h, w), 2.0)
    mf_t = g("mf_t", (b, 128, h, w))
    attn = torch.softmax(g("attn", (b, 1, h * w, h * w), 2.0), -1)
    return sd, net, inp, corr, flow, attn, mf_t


# --------------------------------------------------------------------------------------
# the model
# --------------------------------------------------------------------------------------
def _as_gma(sd: SD, three: bool) -> SD:
    """``update.*`` renamed to GMA's ``update_block.*``; with ``three`` the _sp layers stand in for gru, flow_head and mask."""
    out = {k: v for k, v in sd.items() if not k.startswith("update.")}
    for k, v in sd.items():
        if not k.startswith("update."):
            continue
        k = k[len("update."):]
        for part in ("gru", "flow_head", "mask"):
            if k.startswith(part + "_sp."):
                if not three:
                    k = None
                else:
                    k = part + k[len(part) + 3:]
                break
            if k.startswith(part + ".") and three:
                k = None
                break
        if k is not None:
            out["update_block." + k] = v
    return out


def update(net, inp, corr, flow, attn, sd: SD, mf_t: Optional[Tensor] = None):
    """-> (net, mask, delta_flow, mf).  update.py:109-123 (sd as _as_gma(.., mf_t is not None) gives it)."""
    mf = O.motion_encoder_basic(flow, corr, sd)
    mf_s = G.aggregate(attn, mf, sd)
    x = torch.cat([inp, mf, mf_s] + ([mf_t] if mf_t is not None else []), 1)
    net = O.sep_conv_gru(net, x, sd)
    return net, O.mask_head(net, sd), O.flow_head(net, sd), mf


def forward_one_pair(sd: SD, img1: Tensor, img2: Tensor, iters: int, mf_t: Optional[Tensor] = None):
    """-> (flow_up, mf, low).  splatflow.py:120-154."""
    b = img1.shape[0]
    fmaps = O.encoder(torch.cat([img1, img2], 0), sd, "fnet.", "instance", False)
    fmap1, fmap2 = fmaps[:b], fmaps[b:]
    pyramid = O.corr_pyramid(O.corr_volume(fmap1, fmap2), 4)
    coords0 = O.coords_grid(b, *fmap1.shape[-2:], device=fmap1.device)
    coords1 = coords0.clone()
    cnet = O.encoder(img1, sd, "cnet.", "batch", False)
    net, inp = torch.tanh(cnet[:, :128]), torch.relu(cnet[:, 128:256])
    attn = G.attention(inp, sd, 1)
    g = _as_gma(sd, mf_t is not None)
    mask = mf = None
    for _ in range(iters):
        corr = O.corr_lookup(pyramid, coords1, 4)
        net, mask, delta, mf = update(net, inp, corr, coords1 - coords0, attn, g, mf_t)
        coords1 = coords1 + delta
    low = coords1 - coords0
    return O.convex_upsample(low, mask), mf, low


def splatflow_forward(sd: SD, images: Tensor, iters: int = 32) -> Dict[str, Tensor]:
    """Eval-mode SplatFlow forward (splatflow.py:86-118): pair (0, 1); with three or more frames pair (1, 2) with the splatted mf."""
    sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
    t = images.shape[1]
    x, pads = O.preprocess(images.float())
    flow_up, mf, low = forward_one_pair(sd, x[:, 0], x[:, 1], iters)
    if t > 2:
        flow_up, _, low = forward_one_pair(sd, x[:, 1], x[:, 2], iters, softsplat_average(mf, low))
    return {"flows": O.unpad(flow_up, pads)[:, None], "flow_small": low}


def forward_recipe(recipe: dict, flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with torch.no_grad():
        return splatflow_forward(sd, img, kw.get("iters", 32))
