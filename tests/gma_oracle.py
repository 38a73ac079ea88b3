"""GMA's attention variants on top of the oracle (TEST INFRASTRUCTURE, like oracle/): position-only, position-and-content
and multi-head attention, the aggregate with its projection, the forward loop and the state-dict shapes for any
``num_heads``, plus the synthetic weights and the recipes of the fixtures tests/make_gma_golden.py writes.

Written from the formulas of ptlflow/models/gma/gma_utils.py:6-113 (not from its code) over the building blocks of
oracle/raft_oracle.py.  Notation: N = H*W, d = dim_head = 128, scale s = d^-1/2, P = max_pos_size = 160.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]

MODES = {"content": {}, "position_only": {"position_only": True}, "position_and_content": {"position_and_content": True}}

# end-to-end fixtures: (name, model kwargs, batch, H, W, image kind, weight seed, image seed).  The last one is a ragged image
# (132x164 -> 17x21 grid, N % 8 != 0): the SIMT aggregate of the half-precision path.
E2E_CASES = [
    ("e2e_gma_position_only", dict(iters=6, position_only=True), 1, 128, 192, "smooth", 9, 19),
    ("e2e_gma_position_and_content", dict(iters=6, position_and_content=True), 1, 128, 192, "smooth", 10, 20),
    ("e2e_gma_heads4", dict(iters=6, num_heads=4), 2, 128, 192, "smooth", 11, 21),
    ("e2e_gma_heads2_pc_ragged", dict(iters=6, num_heads=2, position_and_content=True), 1, 132, 164, "noise", 12, 22),
]
E2E = [c[0] for c in E2E_CASES]

# operator fixture op_gma_variants.npz: every mode x heads on two grids, a seeded sample of each output
OP_GRIDS = ((2, 6, 9), (1, 8, 16))  # (batch, H, W): N = 54 (N % 8 != 0) and N = 128
OP_HEADS = (1, 2, 4)
OP_SEED = 72
OP_SAMPLES = 4096
OP_CASES = [(mode, heads, b, h, w) for mode in MODES for heads in OP_HEADS for b, h, w in OP_GRIDS]


def op_sample(numel: int) -> np.ndarray:
    """The seeded subset of an operator output stored in op_gma_variants.npz."""
    return np.sort(np.random.default_rng(2).choice(numel, min(numel, OP_SAMPLES), replace=False))


# --------------------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------------------
def state_dict_shapes(num_heads: int = 1, corr_levels: int = 4, corr_radius: Optional[int] = None) -> Dict[str, Tuple[int, ...]]:
    """O.state_dict_shapes("gma") with heads * d channels in to_qk / to_v and Aggregate.project when heads * d != 128
    (gma.py:100-108, gma_utils.py:41-52, 83-96)."""
    inner = num_heads * 128
    s = {}
    for k, v in O.state_dict_shapes("gma", corr_levels, corr_radius).items():
        if k == "update_block.aggregator.to_v.weight":
            s[k] = (inner, 128, 1, 1)
            if inner != 128:
                s["update_block.aggregator.project.weight"] = (128, inner, 1, 1)
        elif k == "att.to_qk.weight":
            s[k] = (2 * inner, 128, 1, 1)
        else:
            s[k] = v
    return s


def synth_state_dict(shapes, seed: int) -> SD:
    """oracle.synth weights, except that the relative-position tables get nn.Embedding's default N(0, 1) scale: the
    positional logits are then O(1), so a transposed or shifted table index changes the attention far beyond any tolerance
    (synth's generic 0.05 N(0, 1) would keep them near 1e-2)."""
    sd = synth.synth_state_dict(shapes, seed)
    for k, shp in shapes.items():
        if k.endswith(("pos_emb.rel_height.weight", "pos_emb.rel_width.weight")):
            sd[k] = torch.from_numpy(synth.synth_normal(k, shp, seed))
    return sd


def op_inputs(heads: int, b: int, h: int, w: int):
    """(state dict of att.* / update_block.aggregator.*, inp, motion) of one op_gma_variants case, on the CPU."""
    shapes = {k: v for k, v in state_dict_shapes(heads).items()
              if k.startswith(("att.to_qk", "att.pos_emb.rel_h", "att.pos_emb.rel_w", "update_block.aggregator."))}
    sd = synth_state_dict(shapes, OP_SEED + heads)
    inp = torch.relu(torch.from_numpy(synth.synth_normal("gmav/inp", (b, 128, h, w), OP_SEED)))
    motion = torch.from_numpy(synth.synth_normal("gmav/motion", (b, 128, h, w), OP_SEED))
    return sd, inp, motion


def e2e_inputs(recipe):
    """(state_dict, images, kwargs) of an e2e_gma_* fixture."""
    kw = dict(recipe["kwargs"])
    sd = synth_state_dict(state_dict_shapes(kw.get("num_heads", 1)), recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


# --------------------------------------------------------------------------------------
# attention and aggregate
# --------------------------------------------------------------------------------------
def position_logits(q: Tensor, sd: SD, p: str = "att.") -> Tensor:
    """q [B, heads, d, H, W] (already scaled) -> [B, heads, N, N], entry (i = (x, y), j = (u, v)) =
    q(x, y) . E_h[u - x + P - 1] + q(x, y) . E_w[v - y + P - 1]; E_h / E_w = rel_height / rel_width [2P-1, d], one table for
    all heads.  gma_utils.py:6-30."""
    b, heads, d, h, w = q.shape
    eh, ew = sd[p + "pos_emb.rel_height.weight"], sd[p + "pos_emb.rel_width.weight"]
    P = (eh.shape[0] + 1) // 2
    if h > P or w > P:
        raise ValueError(f"{h}x{w} grid exceeds the {P}x{P} relative-position table")
    rh = torch.arange(h, device=q.device)
    rw = torch.arange(w, device=q.device)
    eh_sel = eh[rh[None, :] - rh[:, None] + P - 1]  # [x, u, d]
    ew_sel = ew[rw[None, :] - rw[:, None] + P - 1]  # [y, v, d]
    row = torch.einsum("bkdxy,xud->bkxyu", q, eh_sel)
    col = torch.einsum("bkdxy,yvd->bkxyv", q, ew_sel)
    return (row[..., :, None] + col[..., None, :]).reshape(b, heads, h * w, h * w)


def attention(inp: Tensor, sd: SD, heads: int = 1, position_only: bool = False, position_and_content: bool = False,
              p: str = "att.") -> Tensor:
    """softmax_j(logit_ij) per head -> [B, heads, N, N].  q | k = to_qk(inp), head h = channels h*d ... of each half.
    logit = s q_i . k_j (content), the relative-position term (position_only, which wins when both flags are set), or their
    sum (position_and_content).  gma_utils.py:54-76."""
    b, c, h, w = inp.shape
    qk = F.conv2d(inp, sd[p + "to_qk.weight"])
    d = qk.shape[1] // (2 * heads)
    q = qk[:, : heads * d].reshape(b, heads, d, h, w) * d ** -0.5
    k = qk[:, heads * d :].reshape(b, heads, d, h * w)
    if position_only:
        sim = position_logits(q, sd, p)
    else:
        sim = torch.matmul(q.reshape(b, heads, d, h * w).transpose(2, 3), k)
        if position_and_content:
            sim = sim + position_logits(q, sd, p)
    return torch.softmax(sim, dim=-1)


def aggregate(attn: Tensor, fmap: Tensor, sd: SD, p: str = "update_block.aggregator.") -> Tensor:
    """fmap + gamma * project(concat_h(attn_h @ v_h)), v = to_v(fmap) (head h = channels h*d ...); project only when
    heads * d != C.  attn [B, heads, N, N].  gma_utils.py:79-113."""
    b, c, h, w = fmap.shape
    heads = attn.shape[1]
    v = F.conv2d(fmap, sd[p + "to_v.weight"])
    d = v.shape[1] // heads
    out = torch.matmul(attn, v.reshape(b, heads, d, h * w).transpose(2, 3)).transpose(2, 3).reshape(b, heads * d, h, w)
    if p + "project.weight" in sd:
        out = F.conv2d(out, sd[p + "project.weight"])
    return fmap + sd[p + "gamma"] * out


def update_block(net, inp, corr, flow, attn, sd: SD):
    """-> (net, mask, delta_flow).  gma/update.py:148-160."""
    motion = O.motion_encoder_basic(flow, corr, sd)
    net = O.sep_conv_gru(net, torch.cat([inp, motion, aggregate(attn, motion, sd)], 1), sd)
    return net, O.mask_head(net, sd), O.flow_head(net, sd)


def raft_forward(sd: SD, images: Tensor, iters: int = 12, num_heads: int = 1, position_only: bool = False,
                 position_and_content: bool = False, corr_levels: int = 4, corr_radius: int = 4) -> Dict[str, Tensor]:
    """Eval-mode GMA forward (gma.py:160-222) with any attention mode and number of heads, from the oracle's stages."""
    sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
    x, pads = O.preprocess(images.float())
    img1, img2 = x[:, 0], x[:, 1]
    b = img1.shape[0]
    fmaps = O.encoder(torch.cat([img1, img2], 0), sd, "fnet.", "instance", False)
    fmap1, fmap2 = fmaps[:b], fmaps[b:]
    cnet = O.encoder(img1, sd, "cnet.", "batch", False)
    net, inp = torch.tanh(cnet[:, :128]), torch.relu(cnet[:, 128:256])
    pyramid = O.corr_pyramid(O.corr_volume(fmap1, fmap2), corr_levels)
    coords0 = O.coords_grid(b, *fmap1.shape[-2:], device=fmap1.device)
    coords1 = coords0.clone()
    attn = attention(inp, sd, num_heads, position_only, position_and_content)
    mask = None
    for _ in range(iters):
        corr = O.corr_lookup(pyramid, coords1, corr_radius)
        net, mask, delta = update_block(net, inp, corr, coords1 - coords0, attn, sd)
        coords1 = coords1 + delta
    flow_small = coords1 - coords0
    return {"flows": O.unpad(O.convex_upsample(flow_small, mask), pads)[:, None], "flow_small": flow_small}
