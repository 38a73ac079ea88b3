"""LLA-Flow on top of oracle/raft_oracle.py (TEST INFRASTRUCTURE, like oracle/): the local similarity attention, the local aggregation
of fmap2, the shift-aggregated volume term and the forward, written from their definitions, and the recipes of the fixtures
tests/make_llaflow_golden.py writes.

Written from the formulas of ptlflow/models/llaflow/llaflow.py:140-217, aggregate.py and corr.py, fp32 on the CPU.  delta_l =
(l // 5 - 2, l % 5 - 2) as (dy, dx), clamp() = replicate padding:
  attention: a[n, l] = softmax_l(<q[n], k[clamp(n + delta_l)]> / sqrt(128)), q | k = to_qk(inp) (ls1 and ls2 both on inp)
  LSA:       fmap2' = fmap2 + lsa.gamma sum_l a2[n, l] v[clamp(n + delta_l)], v = lsa.to_v(fmap2)
  volume:    <fmap1[n], fmap2'[m]> / 16 + gamma sum_l a1[n, l] <f1'[clamp(n + delta_l)], f2''[clamp(m + delta_l)]> / 16,
             f1' = s_lsa.to_f1(fmap1), f2'' = s_lsa.to_f2(fmap2'); then RAFT's 4-level pyramid and lookup
  loop:      GMA's (content attention of att.to_qk on inp, one head) for llaflow, RAFT's for llaflow_raft
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
TAPS = 25

# end-to-end fixtures: (name, model, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_llaflow_default", "llaflow", dict(iters=4), 1, 128, 160, "smooth", 411, 421, False),
    ("e2e_llaflow_ragged", "llaflow", dict(iters=3), 2, 129, 131, "noise", 412, 422, False),  # 1/8 grid 17 x 17
    ("e2e_llaflow_warm", "llaflow", dict(iters=3), 1, 128, 160, "smooth", 413, 423, True),
    ("e2e_llaflow_r3", "llaflow", dict(corr_radius=3, iters=3), 1, 128, 136, "smooth", 414, 424, False),
    ("e2e_llaflow_alt", "llaflow", dict(alternate_corr=True, iters=3), 1, 128, 160, "smooth", 415, 425, False),
    ("e2e_llaflow_raft_default", "llaflow_raft", dict(iters=4), 1, 128, 160, "smooth", 416, 426, False),
    ("e2e_llaflow_raft_ragged", "llaflow_raft", dict(iters=3), 2, 129, 131, "noise", 417, 427, False),
    ("e2e_llaflow_raft_warm", "llaflow_raft", dict(iters=3), 1, 128, 160, "smooth", 418, 428, True),
    ("e2e_llaflow_raft_r3", "llaflow_raft", dict(corr_radius=3, iters=3), 1, 136, 128, "smooth", 419, 429, False),
    ("e2e_llaflow_raft_alt", "llaflow_raft", dict(alternate_corr=True, iters=3), 1, 128, 160, "smooth", 420, 430, False),
]
E2E = [c[0] for c in E2E_CASES]
OP_SEED = 431
OP_GRID = (2, 9, 11)  # (batch, H, W) of the operator fixtures: borders on every side, N = 99
OP_ITER_GRID = (8, 8)
# s_lsa.to_f1 and to_f2 are scaled by this factor.  With oracle.synth's unscaled 1x1 weights (variance 1/3 per input channel) the
# gamma corr2 term measured 0.3-4 % of the plain term's max-abs across the fixtures (tests/make_llaflow_golden.py prints it), too
# small to show a wrong shift or a wrong tap order; scaled, the ratios are 0.21-2.8.
SHIFT_SCALE = 8.0


def recipe_of(case) -> dict:
    name, model, kw, b, h, w, kind, ws, iseed, warm = case
    return dict(model=model, kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm)


def state_dict_shapes(model: str = "llaflow", radius: int = 4):
    """The reference's state_dict names and shapes (written by tests/make_llaflow_golden.py for the default radius 4)."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"state_shapes_{model}.json")) as f:
        shapes = {k: tuple(v) for k, v in json.load(f).items()}
    shapes["update_block.encoder.convc1.weight"] = (256, LEVELS * (2 * radius + 1) ** 2, 1, 1)
    return shapes


def synth_state_dict(model: str, radius: int, seed: int) -> SD:
    """oracle.synth's weights with s_lsa.to_f1 / to_f2 scaled by SHIFT_SCALE.  Every scalar ending in ``gamma`` (the volume's gamma,
    lsa.gamma, GMA's aggregator gamma) is 0.5 + 0.1 N(0, 1) there, not the reference's initial 0, so the new terms are visible."""
    sd = synth.synth_state_dict(state_dict_shapes(model, radius), seed)
    for k in ("s_lsa.to_f1.weight", "s_lsa.to_f2.weight"):
        sd[k] = sd[k] * SHIFT_SCALE
    return sd


# --------------------------------------------------------------------------------------
# operators (NCHW)
# --------------------------------------------------------------------------------------
def patches(x: Tensor) -> Tensor:
    """x [B,C,H,W] -> [B,C,25,H,W], tap l = x[clamp(y + l // 5 - 2), clamp(x + l % 5 - 2)]."""
    b, c, h, w = x.shape
    xp = F.pad(x, (2, 2, 2, 2), mode="replicate")
    return torch.stack([xp[:, :, dy:dy + h, dx:dx + w] for dy in range(5) for dx in range(5)], 2)


def local_similar(inp: Tensor, w_qk: Tensor) -> Tensor:
    """-> a [B, H*W, 25]."""
    b, c, h, w = inp.shape
    qk = F.conv2d(inp, w_qk)
    q, k = qk[:, :c], patches(qk[:, c:])
    sim = torch.einsum("bcyx,bclyx->byxl", q * c ** -0.5, k)
    return torch.softmax(sim.reshape(b, h * w, TAPS), dim=-1)


def local_aggregate(a2: Tensor, fmap2: Tensor, sd: SD) -> Tensor:
    b, c, h, w = fmap2.shape
    v = patches(F.conv2d(fmap2, sd["lsa.to_v.weight"]))  # [B,C,25,H,W]
    out = torch.einsum("byxl,bclyx->bcyx", a2.reshape(b, h, w, TAPS), v)
    return fmap2 + sd["lsa.gamma"] * out


def shift_corr(a1: Tensor, fmap1: Tensor, fmap2p: Tensor, sd: SD) -> Tensor:
    """corr2 [B*H*W, 1, H, W] = sum_l a1[n, l] <f1'[clamp(n + delta_l)], f2''[clamp(m + delta_l)]> / 16."""
    b, c, h, w = fmap1.shape
    f1s = patches(F.conv2d(fmap1, sd["s_lsa.to_f1.weight"])).reshape(b, c, TAPS, h * w)
    f2s = patches(F.conv2d(fmap2p, sd["s_lsa.to_f2.weight"])).reshape(b, c, TAPS, h * w)
    f1s = f1s * a1.permute(0, 2, 1)[:, None]
    corr = torch.einsum("bcln,bclm->bnm", f1s, f2s) / c ** 0.5
    return corr.reshape(b * h * w, 1, h, w)


def volume(sd: SD, fmap1: Tensor, fmap2: Tensor, inp: Tensor, trace: Optional[dict] = None):
    """(plain term, gamma corr2) [B*H*W, 1, H, W]; their sum is the volume."""
    wq = sd["ls1.to_qk.weight"], sd["ls2.to_qk.weight"]
    a1, a2 = local_similar(inp, wq[0]), local_similar(inp, wq[1])
    fmap2p = local_aggregate(a2, fmap2, sd)
    plain = O.corr_volume(fmap1, fmap2p)
    extra = sd["gamma"] * shift_corr(a1, fmap1, fmap2p, sd)
    if trace is not None:
        trace.update(a1=a1, a2=a2, fmap2p=fmap2p)
    return plain, extra


def forward(sd: SD, images: Tensor, model: str = "llaflow", radius: int = 4, iters: int = 32, flow_init: Optional[Tensor] = None,
            trace: Optional[dict] = None):
    x, pads = O.preprocess(images)
    b = x.shape[0]
    fm = O.encoder(torch.cat([x[:, 0], x[:, 1]], 0), sd, "fnet.", "instance", False)
    f1, f2 = fm[:b], fm[b:]
    cn = O.encoder(x[:, 0], sd, "cnet.", "batch", False)
    net, inp = torch.tanh(cn[:, :128]), torch.relu(cn[:, 128:])
    plain, extra = volume(sd, f1, f2, inp)
    if trace is not None:
        trace.update(plain=plain, extra=extra)
    pyr = O.corr_pyramid(plain + extra, LEVELS)
    attn = O.gma_attention(inp, sd) if model == "llaflow" else None
    H, W = f1.shape[-2:]
    coords0 = O.coords_grid(b, H, W)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    mask = None
    for _ in range(iters):
        corr = O.corr_lookup(pyr, coords1, radius)
        if attn is not None:
            net, mask, delta = O.gma_update_block(net, inp, corr, coords1 - coords0, attn, sd)
        else:
            net, mask, delta = O.basic_update_block(net, inp, corr, coords1 - coords0, sd)
        coords1 = coords1 + delta
    flows = O.unpad(O.convex_upsample(coords1 - coords0, mask), pads)
    return {"flows": flows[:, None], "flow_small": coords1 - coords0}


def e2e_inputs(recipe):
    kw = dict(recipe["kwargs"])
    sd = synth_state_dict(recipe["model"], kw.get("corr_radius", 4), recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


def forward_recipe(recipe, flow_init: Optional[Tensor] = None, trace: Optional[dict] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(sd, img, recipe["model"], kw.get("corr_radius", 4), kw.get("iters", 32), flow_init, trace)


def op_inputs():
    """Inputs of op_llaflow.npz (llaflow weights, radius 4): features fmap1, fmap2 [2,256,9,11], context inp [2,128,9,11]; one
    update iteration's (net, inp, corr, flow) on an 8x8 grid."""
    sd = synth_state_dict("llaflow", 4, OP_SEED)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    b, h, w = OP_GRID
    hi, wi = OP_ITER_GRID
    x = {
        "fmap1": r("llop/f1", (b, 256, h, w)),
        "fmap2": r("llop/f2", (b, 256, h, w)),
        "inp": torch.relu(r("llop/inp", (b, 128, h, w))),
        "it_net": torch.tanh(r("llop/net", (1, 128, hi, wi))),
        "it_inp": torch.relu(r("llop/itinp", (1, 128, hi, wi))),
        "it_corr": r("llop/corr", (1, LEVELS * 81, hi, wi)),
        "it_flow": r("llop/flow", (1, 2, hi, wi), 3.0),
    }
    return sd, x


def op_outputs(sd: SD, x) -> Dict[str, Tensor]:
    """The oracle's counterpart of make_llaflow_golden.reference_ops."""
    tr: dict = {}
    plain, extra = volume(sd, x["fmap1"], x["fmap2"], x["inp"], tr)
    out = {"a1": tr["a1"], "a2": tr["a2"], "fmap2p": tr["fmap2p"], "volume": plain + extra}
    attn = O.gma_attention(x["it_inp"], sd)
    net, mask, delta = O.gma_update_block(x["it_net"], x["it_inp"], x["it_corr"], x["it_flow"], attn, sd)
    out.update(net=net, mask=mask, delta=delta)
    return out


def np32(t: Tensor) -> np.ndarray:
    return t.detach().float().cpu().numpy().astype(np.float32)
