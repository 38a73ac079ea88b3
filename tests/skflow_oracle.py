"""SKFlow on top of the oracle (TEST INFRASTRUCTURE, like oracle/): the PCBlock, the large-kernel motion encoder, the update block,
the eval forward and the state-dict shapes, plus the recipes of the fixtures tests/make_skflow_golden.py writes.

Written from the formulas of ptlflow/models/skflow/update.py:7-99 and skflow.py:148-232 (not from their code) over the building
blocks of oracle/raft_oracle.py and tests/gma_oracle.py:
  PCBlock(C_in -> C_out, k_conv), h = int(1.5 C_in), GELU = exact erf form:
    x = gelu(x + ffn1(x))                 ffn = 1x1 C_in -> h, GELU, 1x1 h -> C
    x = gelu(x + dw_k(x))  for k in k_conv  (depthwise k x k, zero "same" padding, bias)
    x = gelu(x + pw(x))
    out = ffn2(x)                         (linear)
  motion = cat[conv(cat[convc2(gelu(convc1(corr))), convf2(convf1(flow))]), flow]
  net = gru(cat[net, inp, motion, aggregate(attention, motion)]);  delta = flow_head(net);  mask = 0.25 mask(net)
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

import gma_oracle as GO
from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]

# end-to-end fixtures: (name, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_skflow_default", dict(iters=4), 1, 128, 192, "smooth", 31, 41, False),
    ("e2e_skflow_heads2_pc_ragged", dict(iters=4, num_heads=2, position_and_content=True), 1, 132, 164, "noise", 32, 42, False),
    ("e2e_skflow_warm", dict(iters=4), 1, 128, 192, "smooth", 33, 43, True),
    ("e2e_skflow_altcorr", dict(iters=4, alternate_corr=True), 1, 128, 192, "smooth", 34, 44, False),
    ("e2e_skflow_kconv", dict(iters=5, k_conv=[1, 5, 9], PCUpdater_conv=[3]), 2, 128, 160, "smooth", 35, 45, False),
]
E2E = [c[0] for c in E2E_CASES]

# operator fixture op_skflow.npz: every PCBlock shape of the default model and one update-block iteration, on two grids
OP_GRIDS = ((2, 6, 9), (1, 8, 16))  # 6x9: smaller than the 15x15 kernel, N % 8 != 0
OP_BLOCKS = (("encoder.convc1", 324, 256, "k"), ("encoder.convc2", 256, 192, "k"), ("encoder.convf2", 128, 64, "k"),
             ("encoder.conv", 256, 126, "k"), ("gru", 512, 128, "u"), ("flow_head", 128, 2, "k"))
OP_SEED = 77
OP_SAMPLES = 4096


def op_sample(numel: int) -> np.ndarray:
    """The seeded subset of an operator output stored in op_skflow.npz."""
    return np.sort(np.random.default_rng(3).choice(numel, min(numel, OP_SAMPLES), replace=False))


def gelu(x: Tensor) -> Tensor:
    return 0.5 * x * (1.0 + torch.erf(x * 0.7071067811865476))


# --------------------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------------------
def _pc_shapes(s, p: str, cin: int, cout: int, ks: Sequence[int]) -> None:
    h = int(1.5 * cin)
    for i, k in enumerate(ks):
        s[f"{p}conv_list.{i}.weight"], s[f"{p}conv_list.{i}.bias"] = (cin, 1, k, k), (cin,)
    for name, co, ci in (("ffn1.0", h, cin), ("ffn1.2", cin, h), ("pw", cin, cin), ("ffn2.0", h, cin), ("ffn2.2", cout, h)):
        s[f"{p}{name}.weight"], s[f"{p}{name}.bias"] = (co, ci, 1, 1), (co,)


def state_dict_shapes(k_conv=(1, 15), PCUpdater_conv=(1, 7), num_heads: int = 1, corr_levels: int = 4,
                      corr_radius: int = 4) -> Dict[str, Tuple[int, ...]]:
    """The reference skflow's state_dict names and shapes, in its order (skflow.py:98-121, update.py:44-80)."""
    planes = corr_levels * (2 * corr_radius + 1) ** 2
    s: Dict[str, Tuple[int, ...]] = {k: v for k, v in GO.state_dict_shapes(num_heads, corr_levels, corr_radius).items()
                                     if k.startswith(("fnet.", "cnet."))}
    e = "update_block.encoder."
    _pc_shapes(s, e + "convc1.", planes, 256, k_conv)
    _pc_shapes(s, e + "convc2.", 256, 192, k_conv)
    s[e + "convf1.weight"], s[e + "convf1.bias"] = (128, 2, 1, 1), (128,)
    _pc_shapes(s, e + "convf2.", 128, 64, k_conv)
    _pc_shapes(s, e + "conv.", 256, 126, k_conv)
    _pc_shapes(s, "update_block.gru.", 512, 128, PCUpdater_conv)
    _pc_shapes(s, "update_block.flow_head.", 128, 2, k_conv)
    s["update_block.mask.0.weight"], s["update_block.mask.0.bias"] = (256, 128, 3, 3), (256,)
    s["update_block.mask.2.weight"], s["update_block.mask.2.bias"] = (576, 256, 1, 1), (576,)
    for k, v in GO.state_dict_shapes(num_heads, corr_levels, corr_radius).items():
        if k.startswith(("update_block.aggregator.", "att.")):
            s[k] = v
    return s


def synth_state_dict(shapes, seed: int) -> SD:
    """gma_oracle.synth_state_dict (oracle.synth weights, N(0, 1) position tables)."""
    return GO.synth_state_dict(shapes, seed)


def op_block_inputs(name: str, cin: int, cout: int, kind: str, b: int, h: int, w: int):
    """(state dict of the block with prefix stripped, k_conv, input) of one op_skflow PCBlock case."""
    ks = (1, 7) if kind == "u" else (1, 15)
    shp: Dict[str, Tuple[int, ...]] = {}
    _pc_shapes(shp, "", cin, cout, ks)
    sd = synth.synth_state_dict({f"update_block.{name}.{k}": v for k, v in shp.items()}, OP_SEED)
    sd = {k[len(f"update_block.{name}."):]: v for k, v in sd.items()}
    x = torch.from_numpy(synth.synth_normal(f"skop/{name}", (b, cin, h, w), OP_SEED))
    return sd, ks, x


def op_iter_inputs(b: int, h: int, w: int):
    """(state dict (update_block.* / att.*), net, inp, corr, flow, attention) of the op_skflow update-iteration case."""
    shapes = {k: v for k, v in state_dict_shapes(num_heads=2).items() if k.startswith(("update_block.", "att."))}
    sd = synth_state_dict(shapes, OP_SEED + 1)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    net, inp = torch.tanh(r("skop/net", (b, 128, h, w))), torch.relu(r("skop/inp", (b, 128, h, w)))
    corr, flow = r("skop/corr", (b, 324, h, w)), r("skop/flow", (b, 2, h, w), 3.0)
    attn = GO.attention(inp, sd, 2, position_and_content=True)
    return sd, net, inp, corr, flow, attn


def e2e_inputs(recipe):
    """(state_dict, images, kwargs) of an e2e_skflow_* fixture."""
    kw = dict(recipe["kwargs"])
    shapes = state_dict_shapes(tuple(kw.get("k_conv", (1, 15))), tuple(kw.get("PCUpdater_conv", (1, 7))), kw.get("num_heads", 1))
    sd = synth_state_dict(shapes, recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


# --------------------------------------------------------------------------------------
# blocks
# --------------------------------------------------------------------------------------
def pc_block(x: Tensor, sd: SD, p: str, k_conv: Sequence[int]) -> Tensor:
    """PCBlock4_Deep_nopool_res (update.py:7-41) with parameters sd[p + ...]."""
    def c1(t, name):
        return F.conv2d(t, sd[p + name + ".weight"], sd[p + name + ".bias"])

    x = gelu(x + c1(gelu(c1(x, "ffn1.0")), "ffn1.2"))
    for i, k in enumerate(k_conv):
        x = gelu(x + F.conv2d(x, sd[f"{p}conv_list.{i}.weight"], sd[f"{p}conv_list.{i}.bias"], padding=k // 2, groups=x.shape[1]))
    x = gelu(x + c1(x, "pw"))
    return c1(gelu(c1(x, "ffn2.0")), "ffn2.2")


def motion_encoder(flow: Tensor, corr: Tensor, sd: SD, k_conv, p: str = "update_block.encoder.") -> Tensor:
    """update.py:44-63 -> [B, 128, H, W] = cat[out (126), flow]."""
    cor = gelu(pc_block(corr, sd, p + "convc1.", k_conv))
    cor = pc_block(cor, sd, p + "convc2.", k_conv)
    flo = F.conv2d(flow, sd[p + "convf1.weight"], sd[p + "convf1.bias"])
    flo = pc_block(flo, sd, p + "convf2.", k_conv)
    out = pc_block(torch.cat([cor, flo], 1), sd, p + "conv.", k_conv)
    return torch.cat([out, flow], 1)


def update_block(net, inp, corr, flow, attn, sd: SD, k_conv=(1, 15), PCUpdater_conv=(1, 7)):
    """-> (net, mask, delta_flow).  update.py:81-99."""
    motion = motion_encoder(flow, corr, sd, k_conv)
    mglobal = GO.aggregate(attn, motion, sd)
    net = pc_block(torch.cat([net, inp, motion, mglobal], 1), sd, "update_block.gru.", PCUpdater_conv)
    delta = pc_block(net, sd, "update_block.flow_head.", k_conv)
    return net, O.mask_head(net, sd), delta


def raft_forward(sd: SD, images: Tensor, iters: int = 12, k_conv=(1, 15), PCUpdater_conv=(1, 7), num_heads: int = 1,
                 position_only: bool = False, position_and_content: bool = False, alternate_corr: bool = False,
                 corr_levels: int = 4, corr_radius: int = 4, flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """Eval-mode SKFlow forward (skflow.py:148-232); flow_init: the forward-interpolated previous flow_small (warm start)."""
    sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
    x, pads = O.preprocess(images.float())
    img1, img2 = x[:, 0], x[:, 1]
    b = img1.shape[0]
    fmaps = O.encoder(torch.cat([img1, img2], 0), sd, "fnet.", "instance", False)
    fmap1, fmap2 = fmaps[:b], fmaps[b:]
    cnet = O.encoder(img1, sd, "cnet.", "batch", False)
    net, inp = torch.tanh(cnet[:, :128]), torch.relu(cnet[:, 128:256])
    pyramid = None if alternate_corr else O.corr_pyramid(O.corr_volume(fmap1, fmap2), corr_levels)
    coords0 = O.coords_grid(b, *fmap1.shape[-2:], device=fmap1.device)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    attn = GO.attention(inp, sd, num_heads, position_only, position_and_content)
    mask = None
    for _ in range(iters):
        if alternate_corr:
            corr = O.alt_corr_lookup(fmap1, fmap2, coords1, corr_radius, corr_levels)
        else:
            corr = O.corr_lookup(pyramid, coords1, corr_radius)
        net, mask, delta = update_block(net, inp, corr, coords1 - coords0, attn, sd, k_conv, PCUpdater_conv)
        coords1 = coords1 + delta
    flow_small = coords1 - coords0
    return {"flows": O.unpad(O.convex_upsample(flow_small, mask), pads)[:, None], "flow_small": flow_small}
