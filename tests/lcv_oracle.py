"""LCV on top of oracle/raft_oracle.py (TEST INFRASTRUCTURE, like oracle/): the learned bilinear form, the pyramid that stops pooling,
its lookup and the forward, written from their definitions, and the recipes of the fixtures tests/make_lcv_golden.py writes.

Written from the formulas of ptlflow/models/lcv/corr_lcv.py and lcv_raft.py, fp32 on the CPU:
  fold:     S = (triu(raw_P) - triu(raw_P)^T) / 2, P = (eye + S)(eye - S)^-1, t = atan(raw_D) 2 / pi, D = diag((1 + t) / (1 - t)),
            W = P^T D P (corr_lcv.py:19-31)
  volume:   <f1^T W, f2> / sqrt(C) from the fp32 features (lcv_raft.py:145-147, corr_lcv.py:33-39)
  pyramid:  level l is the 2x2 mean of level l-1 while the smaller side of level l-1 exceeds 2r+1, else level l-1 again
            (corr_lcv.py:44-50); the lookup samples level l at coords / 2^l whatever its size (corr_lcv.py:52-75)
  frames:   BGR, not swapped (lcv_raft.py:126-134, bgr_to_rgb=False), else RAFT's pre-processing
  loop:     RAFT's BasicUpdateBlock + convex 8x upsample (lcv_raft), or SmallUpdateBlock + upflow8 (lcv_raft_small)
"""
from __future__ import annotations

import json
import math
import os
from typing import Dict, List, Optional, Tuple

import torch

from oracle import raft_oracle as O
from oracle import synth
from oracle.fixtures import images

Tensor = torch.Tensor
SD = Dict[str, Tensor]
HERE = os.path.dirname(os.path.abspath(__file__))

# end-to-end fixtures: (name, model, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_lcv_raft_pooling", "lcv_raft", dict(iters=3), 1, 320, 384, "smooth", 411, 421, False),  # 40x48: every level pools
    ("e2e_lcv_raft_ragged", "lcv_raft", dict(iters=3), 1, 131, 165, "noise", 412, 422, False),  # 17x21, 8x10, 8x10, 8x10
    ("e2e_lcv_raft_never", "lcv_raft", dict(iters=3), 1, 64, 64, "smooth", 413, 423, False),  # 8x8 never pools
    ("e2e_lcv_raft_tiny", "lcv_raft", dict(iters=3), 1, 32, 32, "smooth", 414, 424, False),  # 4x4: raft's pyramid would be empty
    ("e2e_lcv_raft_b2", "lcv_raft", dict(iters=3), 2, 96, 128, "noise", 415, 425, False),  # 12x16, 6x8, 6x8, 6x8
    ("e2e_lcv_raft_warm", "lcv_raft", dict(iters=3), 1, 128, 160, "smooth", 416, 426, True),
    ("e2e_lcv_raft_r3l3", "lcv_raft", dict(corr_radius=3, corr_levels=3, iters=3), 1, 128, 160, "smooth", 417, 427, False),
    ("e2e_lcv_raft_small_default", "lcv_raft_small", dict(iters=3), 1, 128, 160, "smooth", 418, 428, False),
    ("e2e_lcv_raft_small_ragged", "lcv_raft_small", dict(iters=3), 2, 131, 165, "noise", 419, 429, False),
]
E2E = [c[0] for c in E2E_CASES]
# the learned form's recipe: raw_P = eye + N(0, P_SCALE^2) upper triangle, raw_D ~ N(0, D_SCALE^2), so that W is far from the
# identity of the reference's initialisation (with W = I and an all-pooling grid LCV is RAFT, and a fixture would not test W)
P_SCALE, D_SCALE = 0.3, 0.5
OP_SEED = 431
OP_DIM, OP_GRID, OP_RADIUS, OP_LEVELS = 64, (12, 13), 4, 4  # levels 12x13, 6x6, 6x6, 6x6


def recipe_of(case) -> dict:
    name, model, kw, b, h, w, kind, ws, iseed, warm = case
    return dict(model=model, kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm)


def state_dict_shapes(model: str = "lcv_raft", corr_levels: int = 4, corr_radius: Optional[int] = None) -> Dict[str, Tuple[int, ...]]:
    """The reference's state_dict names and shapes (written by tests/make_lcv_golden.py for the default hparams)."""
    with open(os.path.join(HERE, "golden", f"state_shapes_{model}.json")) as f:
        shapes = {k: tuple(v) for k, v in json.load(f).items()}
    r = corr_radius if corr_radius is not None else (4 if model == "lcv_raft" else 3)
    convc1 = shapes["update_block.encoder.convc1.weight"]
    shapes["update_block.encoder.convc1.weight"] = (convc1[0], corr_levels * (2 * r + 1) ** 2, 1, 1)
    return shapes


def learned_form(dim: int, seed: int) -> SD:
    """raw_P, raw_D and eye of the recipe (see P_SCALE, D_SCALE)."""
    up = torch.triu(torch.from_numpy(synth.synth_normal("lcv.raw_P", (dim, dim), seed, P_SCALE)))
    return {"raw_P": torch.eye(dim) + up, "raw_D": torch.from_numpy(synth.synth_normal("lcv.raw_D", (dim,), seed, D_SCALE)),
            "eye": torch.eye(dim)}


def synth_state_dict(model: str, seed: int, corr_levels: int = 4, corr_radius: Optional[int] = None) -> SD:
    sd = synth.synth_state_dict(state_dict_shapes(model, corr_levels, corr_radius), seed)
    dim = sd["corr_block.raw_D"].shape[0]
    sd.update({"corr_block." + k: v for k, v in learned_form(dim, seed).items()})
    return sd


# --------------------------------------------------------------------------------------
# operators
# --------------------------------------------------------------------------------------
def bilinear_form(raw_P: Tensor, raw_D: Tensor, eye: Tensor) -> Tensor:
    up = torch.triu(raw_P)
    S = (up - up.t()) / 2
    P = (eye + S) @ torch.inverse(eye - S)
    t = torch.atan(raw_D) * 2 / math.pi
    return P.t() @ torch.diag((1 + t) / (1 - t)) @ P


def level_sizes(h: int, w: int, levels: int, radius: int) -> List[Tuple[int, int]]:
    sizes = [(h, w)]
    for _ in range(levels - 1):
        ph, pw = sizes[-1]
        sizes.append((ph // 2, pw // 2) if min(ph, pw) > 2 * radius + 1 else (ph, pw))
    return sizes


def volume(f1: Tensor, f2: Tensor, W: Tensor) -> Tensor:
    """f [B,C,H,W] -> [B*H*W, 1, H, W] = <f1^T W, f2> / sqrt(C)."""
    b, c, h, w = f1.shape
    a = torch.einsum("bcn,cd->bnd", f1.reshape(b, c, h * w), W)
    return (torch.bmm(a, f2.reshape(b, c, h * w)) / math.sqrt(c)).reshape(b * h * w, 1, h, w)


def pyramid(vol: Tensor, levels: int, radius: int) -> List[Tensor]:
    pyr = [vol]
    for _ in range(levels - 1):
        v = pyr[-1]
        pyr.append(O.corr_pyramid(v, 2)[1] if min(v.shape[-2:]) > 2 * radius + 1 else v)
    return pyr


def forward(sd: SD, images_: Tensor, model: str = "lcv_raft", iters: int = 32, corr_levels: int = 4, corr_radius: Optional[int] = None,
            flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    small = model == "lcv_raft_small"
    radius = corr_radius if corr_radius is not None else (3 if small else 4)
    hdim, cdim = (96, 64) if small else (128, 128)
    sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
    x, pads = O.preprocess(images_.float().flip(-3))  # O.preprocess swaps BGR -> RGB; LCV keeps BGR
    img1, img2 = x[:, 0], x[:, 1]
    b = img1.shape[0]
    fmaps = O.encoder(torch.cat([img1, img2], 0), sd, "fnet.", "instance", small)
    fmap1, fmap2 = fmaps[:b], fmaps[b:]
    cnet = O.encoder(img1, sd, "cnet.", "none" if small else "batch", small)
    net, inp = torch.tanh(cnet[:, :hdim]), torch.relu(cnet[:, hdim: hdim + cdim])
    W = bilinear_form(sd["corr_block.raw_P"], sd["corr_block.raw_D"], sd["corr_block.eye"])
    pyr = pyramid(volume(fmap1, fmap2, W), corr_levels, radius)
    h8, w8 = fmap1.shape[-2:]
    coords0 = O.coords_grid(b, h8, w8)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    block = O.small_update_block if small else O.basic_update_block
    mask = None
    for _ in range(iters):
        corr = O.corr_lookup(pyr, coords1, radius)
        net, mask, delta = block(net, inp, corr, coords1 - coords0, sd)
        coords1 = coords1 + delta
    flow_small = coords1 - coords0
    up = O.upflow8(flow_small) if mask is None else O.convex_upsample(flow_small, mask)
    return {"flows": O.unpad(up, pads)[:, None], "flow_small": flow_small}


def e2e_inputs(recipe):
    kw = dict(recipe["kwargs"])
    sd = synth_state_dict(recipe["model"], recipe["wseed"], kw.get("corr_levels", 4), kw.get("corr_radius"))
    return sd, images(recipe), kw


def forward_recipe(recipe, flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(sd, img, recipe["model"], kw.get("iters", 32), kw.get("corr_levels", 4), kw.get("corr_radius"), flow_init)


def op_inputs():
    """(learned form of OP_DIM, f1, f2 [1, OP_DIM, *OP_GRID], coords [1, 2, *OP_GRID] spread past the frozen levels' borders)."""
    h, w = OP_GRID
    form = learned_form(OP_DIM, OP_SEED)
    f1 = torch.from_numpy(synth.synth_normal("lcv.op.f1", (1, OP_DIM, h, w), OP_SEED))
    f2 = torch.from_numpy(synth.synth_normal("lcv.op.f2", (1, OP_DIM, h, w), OP_SEED))
    coords = O.coords_grid(1, h, w) + torch.from_numpy(synth.synth_normal("lcv.op.coords", (1, 2, h, w), OP_SEED, 4.0))
    return form, f1, f2, coords


def op_outputs() -> Dict[str, Tensor]:
    form, f1, f2, coords = op_inputs()
    W = bilinear_form(form["raw_P"], form["raw_D"], form["eye"])
    pyr = pyramid(volume(f1, f2, W), OP_LEVELS, OP_RADIUS)
    return {"W": W, "level_sizes": torch.tensor([tuple(p.shape[-2:]) for p in pyr], dtype=torch.float32),
            "lookup": O.corr_lookup(pyr, coords, OP_RADIUS)}
