"""SCV on top of oracle/raft_oracle.py (TEST INFRASTRUCTURE, like oracle/): the encoders with projected shortcuts, the exact k-NN, the
sparse pyramid splat, the convex 4x and the forward, written from their definitions, and the recipes of the fixtures
tests/make_scv_golden.py writes.

Written from the formulas of ptlflow/models/scv/, fp32 on the CPU:
  encoders: RAFT's BasicEncoder with a 1x1 conv + norm shortcut in every residual block, stage strides 1, 2, 2 (scv8) or 1, 2, 1 (scv4)
            (extractor.py:6-270)
  k-NN:     scores <f1[q], f2[t]> in float64, the num_k largest per query (ties to the lower target); the kept value is the fp32
            <f1[q], f2[t]> / sqrt(C) (scv.py:48-83)
  lookup:   displacement d = (ty - qy, tx - qx) - sum of the deltas so far; for level i the bilinear corners of d / 2^i with both
            coordinates in [-4, 4] add weight * value to bin i * 81 + (cy + 4) * 9 + (cx + 4) -- explicit loops over matches, levels and
            corners, no torch.sparse (scv.py:248-298, utils.py:148-175)
  loop:     RAFT's BasicUpdateBlock over the 405 bins, convex 8x (scv8) or 4x of 4 * flow (scv4, scv.py:186-197)
"""
from __future__ import annotations

import json
import math
import os
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]
LEVELS, RANGE = 5, 4
PLANES = LEVELS * 81
MODELS = ("scv4", "scv8")
STRIDES = {"scv4": (1, 2, 1), "scv8": (1, 2, 2)}
UPSAMPLE = {"scv4": 4, "scv8": 8}

# end-to-end fixtures: (name, model, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_scv8_default", "scv8", dict(iters=3), 1, 96, 128, "smooth", 411, 421, False),
    ("e2e_scv8_k8", "scv8", dict(num_k=8, iters=3), 1, 96, 128, "smooth", 412, 422, False),
    ("e2e_scv8_ragged", "scv8", dict(iters=2), 1, 83, 117, "noise", 413, 423, False),
    ("e2e_scv8_b2", "scv8", dict(iters=2), 2, 64, 96, "smooth", 414, 434, False),
    ("e2e_scv8_warm", "scv8", dict(iters=2), 1, 96, 128, "smooth", 415, 425, True),
    ("e2e_scv4_default", "scv4", dict(iters=3), 1, 64, 96, "smooth", 416, 426, False),
    ("e2e_scv4_k8", "scv4", dict(num_k=8, iters=3), 1, 64, 96, "smooth", 417, 427, False),
    ("e2e_scv4_ragged", "scv4", dict(iters=2), 1, 61, 75, "noise", 418, 428, False),
    ("e2e_scv4_b2", "scv4", dict(iters=2), 2, 48, 64, "smooth", 419, 439, False),
    ("e2e_scv4_warm", "scv4", dict(iters=2), 1, 64, 96, "smooth", 420, 440, True),
]
E2E = [c[0] for c in E2E_CASES]
OP_SEED = 431
OP_KNN = dict(B=1, H=9, W=11, C=256, k=32)  # the k-NN operator: N = 99 queries and targets
OP_ITER_GRID = (8, 8)


def recipe_of(case) -> dict:
    name, model, kw, b, h, w, kind, ws, iseed, warm = case
    return dict(model=model, kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm)


def state_dict_shapes(model: str):
    """The reference's state_dict names and shapes (written by tests/make_scv_golden.py)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"state_shapes_{model}.json")) as f:
        return {k: tuple(v) for k, v in json.load(f).items()}


def synth_state_dict(model: str, seed: int) -> SD:
    return synth.synth_state_dict(state_dict_shapes(model), seed)


# --------------------------------------------------------------------------------------
# operators
# --------------------------------------------------------------------------------------
def _block(x: Tensor, sd: SD, p: str, kind: str, stride: int) -> Tensor:
    y = torch.relu(O._norm(O._conv(x, sd, p + "conv1", stride=stride, padding=1), sd, p + "norm1", kind))
    y = torch.relu(O._norm(O._conv(y, sd, p + "conv2", padding=1), sd, p + "norm2", kind))
    x = O._norm(O._conv(x, sd, p + "downsample.0", stride=stride), sd, p + "downsample.1", kind)  # always projected
    return torch.relu(x + y)


def encoder(x: Tensor, sd: SD, prefix: str, kind: str, strides) -> Tensor:
    x = torch.relu(O._norm(O._conv(x, sd, prefix + "conv1", stride=2, padding=3), sd, prefix + "norm1", kind))
    for li, stride in enumerate(strides, start=1):
        x = _block(x, sd, f"{prefix}layer{li}.0.", kind, stride)
        x = _block(x, sd, f"{prefix}layer{li}.1.", kind, 1)
    return O._conv(x, sd, prefix + "conv2")


def knn(f1: Tensor, f2: Tensor, k: int):
    """f1, f2 [B,C,H,W] -> (val fp32 [B,N,k], idx int64 [B,N,k], gap): the exact top-k of the float64 scores, descending, ties to the
    lower target; val is the fp32 score / sqrt(C) of the reference; gap is the smallest float64 distance between the k-th and the
    (k+1)-th score of any query (inf when k = N)."""
    b, c, h, w = f1.shape
    a, t = f1.reshape(b, c, -1).double(), f2.reshape(b, c, -1).double()
    s = torch.einsum("bcn,bcm->bnm", a, t)
    n = s.shape[-1]
    order = torch.argsort(-s, dim=-1, stable=True)  # stable: equal scores keep the lower target first
    idx = order[..., :k]
    srt = torch.gather(s, -1, order)
    gap = float((srt[..., k - 1] - srt[..., k]).min()) if k < n else math.inf
    g = torch.gather(f2.reshape(b, c, 1, -1).expand(b, c, f1.shape[2] * f1.shape[3], n).float(), 3,
                     idx.unsqueeze(1).expand(b, c, -1, -1))  # [B, C, N, k]
    val = torch.einsum("bcn,bcnk->bnk", f1.reshape(b, c, -1).float(), g) / math.sqrt(c)
    return val, idx, gap


def displacements(idx: Tensor, h: int, w: int) -> Tensor:
    """idx [B,N,k] -> the reference's coords1_cv at iteration 0: (ty - qy, tx - qx) fp32 [B,N,k,2]."""
    n = torch.arange(h * w)
    qy, qx = (n // w).view(1, -1, 1), (n % w).view(1, -1, 1)
    return torch.stack([(idx // w - qy).float(), (idx % w - qx).float()], dim=-1)


def splat(disp: Tensor, val: Tensor) -> Tensor:
    """disp fp32 [B,N,k,2] (y, x), val fp32 [B,N,k] -> [B,N,405]: explicit loops over matches, levels and corners."""
    b, n, k, _ = disp.shape
    out = torch.zeros(b, n, PLANES, dtype=torch.float32)
    d, v = disp.reshape(-1, k, 2), val.reshape(-1, k)
    o = out.view(-1, PLANES)
    for j in range(k):
        for lvl in range(LEVELS):
            y, x = d[:, j, 0] * 0.5**lvl, d[:, j, 1] * 0.5**lvl
            yf, xf = torch.floor(y), torch.floor(x)
            yc, xc = yf + 1, xf + 1
            corners = (((yc - y) * (xc - x), yf, xf), ((y - yf) * (xc - x), yc, xf), ((yc - y) * (x - xf), yf, xc),
                       ((y - yf) * (x - xf), yc, xc))
            for wt, cy, cx in corners:
                keep = (cy.abs() <= RANGE) & (cx.abs() <= RANGE)
                rows = keep.nonzero().flatten()
                bins = lvl * 81 + (cy[rows].long() + RANGE) * 9 + (cx[rows].long() + RANGE)
                o[rows, bins] += wt[rows] * v[rows, j]
    return out


def lookup(disp: Tensor, val: Tensor, h: int, w: int) -> Tensor:
    """-> corr [B,405,H,W] as the update block reads it."""
    b = disp.shape[0]
    return splat(disp, val).view(b, h, w, PLANES).permute(0, 3, 1, 2).contiguous()


def convex_upsample4(flow: Tensor, mask: Tensor) -> Tensor:
    """flow [B,2,H,W], mask [B,144,H,W] -> [B,2,4H,4W], the convex 4x of 4 * flow (scv.py:186-197), mask channel = tap * 16 + sy * 4 + sx."""
    b, _, h, w = flow.shape
    m = torch.softmax(mask.view(b, 9, 4, 4, h, w), dim=1)
    f = F.pad(4.0 * flow, (1, 1, 1, 1))
    out = torch.zeros(b, 2, 4, 4, h, w, dtype=flow.dtype)
    for tap in range(9):
        dy, dx = tap // 3, tap % 3
        out = out + m[:, tap][:, None] * f[:, :, dy : dy + h, dx : dx + w][:, :, None, None]
    return out.permute(0, 1, 4, 2, 5, 3).reshape(b, 2, 4 * h, 4 * w)


def forward(model: str, sd: SD, images: Tensor, num_k: int = 32, iters: int = 32, flow_init: Optional[Tensor] = None,
            trace: Optional[dict] = None):
    x, pads = O.preprocess(images)
    b = x.shape[0]
    fm = encoder(torch.cat([x[:, 0], x[:, 1]], 0), sd, "fnet.", "instance", STRIDES[model])
    f1, f2 = fm[:b], fm[b:]
    cn = encoder(x[:, 0], sd, "cnet.", "batch", STRIDES[model])
    net, inp = torch.tanh(cn[:, :128]), torch.relu(cn[:, 128:])
    H, W = f1.shape[-2:]
    val, idx, gap = knn(f1, f2, num_k)
    if trace is not None:
        absdot = torch.einsum("bcn,bcm->bnm", f1.reshape(b, f1.shape[1], -1).abs().double(), f2.reshape(b, f1.shape[1], -1).abs().double())
        trace.update(knn_gap=gap, absdot_max=float(absdot.max()), channels=f1.shape[1])
    disp = displacements(idx, H, W)
    coords0 = O.coords_grid(b, H, W)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    mask = None
    delta = torch.zeros_like(coords0)
    for _ in range(iters):
        disp = disp - delta.permute(0, 2, 3, 1).reshape(b, H * W, 1, 2)[..., [1, 0]]
        net, mask, delta = O.basic_update_block(net, inp, lookup(disp, val, H, W), coords1 - coords0, sd)
        coords1 = coords1 + delta
    up = O.convex_upsample(coords1 - coords0, mask) if model == "scv8" else convex_upsample4(coords1 - coords0, mask)
    return {"flows": O.unpad(up, pads)[:, None], "flow_small": coords1 - coords0}


def e2e_inputs(recipe):
    sd = synth_state_dict(recipe["model"], recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, dict(recipe["kwargs"])


def forward_recipe(recipe, flow_init: Optional[Tensor] = None, trace: Optional[dict] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(recipe["model"], sd, img, kw.get("num_k", 32), kw.get("iters", 32), flow_init, trace)


def op_inputs():
    """Inputs of op_scv.npz: seeded features for the k-NN; displacements and values for the lookup, with entries on and across the
    +-4 edge of every level; one update iteration's (net, inp, corr, flow) per model on an 8 x 8 grid (weights of both models)."""
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    p = OP_KNN
    x = {"f1": r("scvop/f1", (p["B"], p["C"], p["H"], p["W"])), "f2": r("scvop/f2", (p["B"], p["C"], p["H"], p["W"]))}
    n, k = 64, 32
    disp = r("scvop/disp", (1, n, k, 2), 20.0)
    edges = torch.tensor([4.0, -4.0, 4.5, -4.5, 3.999, -4.001, 8.0, -8.0, 9.0, 16.0, -16.0, 17.5, 32.0, -33.0, 64.0, -64.5, 70.0, 0.0])
    disp[0, : edges.numel(), 0, 0] = edges
    disp[0, : edges.numel(), 1, 1] = edges
    disp[0, : edges.numel(), 2] = edges[:, None]
    x["disp"], x["val"] = disp, r("scvop/val", (1, n, k))
    hi, wi = OP_ITER_GRID
    x.update(net=torch.tanh(r("scvop/net", (1, 128, hi, wi))), inp=torch.relu(r("scvop/inp", (1, 128, hi, wi))),
             corr=r("scvop/corr", (1, PLANES, hi, wi)), flow=r("scvop/flow", (1, 2, hi, wi), 3.0))
    sds = {m: synth_state_dict(m, OP_SEED) for m in MODELS}
    return sds, x


def op_outputs(sds, x) -> Dict[str, Tensor]:
    """The oracle's counterpart of make_scv_golden.reference_ops."""
    val, idx, _ = knn(x["f1"], x["f2"], OP_KNN["k"])
    out = {"knn_val": val, "knn_idx": idx, "lookup": splat(x["disp"], x["val"])}
    for m in MODELS:
        net, mask, delta = O.basic_update_block(x["net"], x["inp"], x["corr"], x["flow"], sds[m])
        out.update({f"{m}_net": net, f"{m}_mask": mask, f"{m}_delta": delta})
    return out


def np32(t: Tensor) -> np.ndarray:
    return t.detach().float().cpu().numpy().astype(np.float32)
