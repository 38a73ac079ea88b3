"""CRAFT on top of oracle/raft_oracle.py (TEST INFRASTRUCTURE, like oracle/): the three cross-attention sites, the globally
normalised inter-frame volume and the forward, written from their definitions, and the recipes of the fixtures
tests/make_craft_golden.py writes.

Written from the formulas of ptlflow/models/craft/craft.py:269-376, setrans.py:320-926, corr.py:141-218 and update.py:131-196, fp32 on
the CPU.  Tokens are pixel-major [B, N, C], N = H*W, query i at (qy, qx) = divmod(i, W), key j at (ky, kx):
  LN(x)      = LayerNorm over channels, eps 1e-12, no affine
  scores_m   = q_m . k_m / sqrt(C / M), q = LN(x1) Wq^T (+ b), k = LN(x2) Wk^T (+ b), modes of C / M channels
  clamp      = clamp(-100, 100) of every score when the largest score of the call exceeds 100 (all samples and modes)
  bias(i, j) = w_pos biases[ky - qy + R][kx - qx + R] when both offsets are within R, else 0
  f2 trans   = LN(coeff x + sum_m softmax_m(<w, y_m>) y_m), y_m = softmax_j(clamp(scores_m) + bias (- 1e9 outside the mask)) V_m,
               x = LN(fmap2), V = x first_linear^T
  volume     = LN over the N^2 values of sum_m softmax_m(a s_m) s_m, s_m = clamp(scores_m) + bias, of LN(fmap1) and LN(f2 trans)
               with the shared q = k projection; then RAFT's 4-level pyramid (craft=False: RAFT's volume of fmap1 and f2 trans)
  loop       = GMA's, with motion_global = the aggregator (as the f2 trans, on the motion features) of the intra-frame probabilities
"""
from __future__ import annotations

import json
import os
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth
from oracle.fixtures import images

Tensor = torch.Tensor
SD = Dict[str, Tensor]
LEVELS = 4
CLIP = 100.0
# synth's rank-2 weights are 0.05 N(0, 1); these entries are scaled so that the position biases and the mode scores matter
BIAS_SCALE = 20.0
SCORE_SCALE = 20.0

# end-to-end fixtures: (name, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start, query scale)
E2E_CASES = [
    ("e2e_craft_default", dict(iters=4), 1, 128, 160, "smooth", 511, 521, False, 1.0),
    ("e2e_craft_ragged", dict(iters=3), 1, 129, 131, "noise", 512, 522, False, 1.0),  # 1/8 grid 17 x 17
    ("e2e_craft_b2", dict(iters=3), 2, 128, 144, "smooth", 513, 523, False, 1.0),
    ("e2e_craft_warm", dict(iters=3), 1, 128, 160, "smooth", 514, 524, True, 1.0),
    ("e2e_craft_nocraft", dict(craft=False, iters=3), 1, 128, 160, "smooth", 515, 525, False, 1.0),
    ("e2e_craft_modes", dict(inter_num_modes=2, intra_num_modes=1, f2_num_modes=2, pos_bias_radius=3, corr_radius=3, iters=3), 1, 128, 136,
     "smooth", 516, 526, False, 1.0),
    ("e2e_craft_mask", dict(f2_attn_mask_radius=4, iters=3), 1, 128, 160, "smooth", 517, 527, False, 1.0),
    # the inter-frame query weights scaled so that exactly one sample of the pair exceeds the clip (tests/test_craft.py checks it)
    ("e2e_craft_clamp", dict(iters=3), 2, 128, 144, "smooth", 518, 528, False, 3.889),
]
E2E = [c[0] for c in E2E_CASES]


def recipe_of(case) -> dict:
    name, kw, b, h, w, kind, ws, iseed, warm, qscale = case
    return dict(model="craft", kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm, qscale=qscale)


def state_dict_shapes(kw: Optional[dict] = None):
    """The reference's state_dict names and shapes for the constructor keywords ``kw`` (from the default model's, written by
    tests/make_craft_golden.py)."""
    kw = kw or {}
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "state_shapes_craft.json")) as f:
        shapes = {k: tuple(v) for k, v in json.load(f).items()}
    r = kw.get("corr_radius", 4)
    R = kw.get("pos_bias_radius", 7)
    shapes["update_block.encoder.convc1.weight"] = (256, LEVELS * (2 * r + 1) ** 2, 1, 1)
    modes = {"corr_fn": kw.get("inter_num_modes", 4), "att": kw.get("intra_num_modes", 4)}
    for k in list(shapes):
        if k.endswith("pos_coder.biases"):
            shapes[k] = (2 * R + 1, 2 * R + 1)
        for p, m in modes.items():
            if k.startswith(p + ".setrans.attn_softaggr") and m == 1:
                del shapes[k]
    shapes["f2_trans.setrans.out_trans.first_linear.weight"] = (256 * kw.get("f2_num_modes", 4), 256)
    shapes["update_block.aggregator.first_linear.weight"] = (128 * kw.get("intra_num_modes", 4), 128)
    if not kw.get("craft", True):
        shapes = {k: v for k, v in shapes.items() if not k.startswith("corr_fn.")}
    return shapes


def synth_state_dict(kw: dict, seed: int, qscale: float = 1.0) -> SD:
    """oracle.synth's weights with the position biases and the feat2score weights scaled (BIAS_SCALE, SCORE_SCALE), every
    input_skip_coeff 1 + that, the inter-frame key equal to its query (the reference ties them) and both scaled by ``qscale``."""
    sd = synth.synth_state_dict(state_dict_shapes(kw), seed)
    for k in list(sd):
        if k.endswith("pos_coder.biases"):
            sd[k] = sd[k] * BIAS_SCALE
        elif k.endswith("feat2score.weight"):
            sd[k] = sd[k] * SCORE_SCALE
        elif k.endswith("input_skip_coeff"):
            sd[k] = 1.0 + sd[k]
    if "corr_fn.setrans.query.weight" in sd:
        for s in ("weight", "bias"):
            if "corr_fn.setrans.query." + s in sd:
                sd["corr_fn.setrans.query." + s] = sd["corr_fn.setrans.query." + s] * qscale
                sd["corr_fn.setrans.key." + s] = sd["corr_fn.setrans.query." + s].clone()
    return sd


# --------------------------------------------------------------------------------------
# operators (tokens [B, N, C])
# --------------------------------------------------------------------------------------
def ln(x: Tensor) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), eps=1e-12)


def tokens(x: Tensor) -> Tensor:
    b, c, h, w = x.shape
    return x.reshape(b, c, h * w).transpose(1, 2)


def window_bias(biases: Tensor, H: int, W: int) -> Tensor:
    """[N, N]: biases[ky - qy + R][kx - qx + R] inside the window, 0 outside."""
    R = (biases.shape[0] - 1) // 2
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    ys, xs = ys.reshape(-1), xs.reshape(-1)
    dy, dx = ys[None, :] - ys[:, None], xs[None, :] - xs[:, None]
    inside = (dy.abs() <= R) & (dx.abs() <= R)
    return torch.where(inside, biases[(dy + R).clamp(0, 2 * R), (dx + R).clamp(0, 2 * R)], torch.zeros((), dtype=biases.dtype))


def chebyshev_mask(H: int, W: int, radius: int) -> Tensor:
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    ys, xs = ys.reshape(-1), xs.reshape(-1)
    far = torch.maximum((ys[None, :] - ys[:, None]).abs(), (xs[None, :] - xs[:, None]).abs()) > radius
    return far.float() * -1e9


def mode_scores(x1: Tensor, x2: Tensor, sd: SD, p: str, M: int) -> Tensor:
    """[B, M, N1, N2] = q_m . k_m / sqrt(C / M)."""
    b, n1, c = x1.shape
    d = c // M
    q = F.linear(x1, sd[p + "query.weight"], sd.get(p + "query.bias"))
    k = F.linear(x2, sd[p + "key.weight"], sd.get(p + "key.bias"))
    q = q.view(b, n1, M, d).transpose(1, 2)
    k = k.view(b, x2.shape[1], M, d).transpose(1, 2)
    return q @ k.transpose(-1, -2) / d ** 0.5


def clamp(s: Tensor) -> Tensor:
    return s.clamp(-CLIP, CLIP) if s.max().item() > CLIP else s


def probs(x: Tensor, sd: SD, p: str, M: int, w_pos: float, H: int, W: int, mask_radius: int = -1) -> Tensor:
    """SelfAttVisPosTrans's attention probabilities of the tokens x [B, N, C]: [B, M, N, N]."""
    s = clamp(mode_scores(ln(x), ln(x), sd, p + "setrans.", M)) + w_pos * window_bias(sd[p + "vispos_encoder.pos_coder.biases"], H, W)
    if mask_radius > 0:
        s = s + chebyshev_mask(H, W, mask_radius)
    return torch.softmax(s, dim=-1)


def expanded(x: Tensor, attn: Tensor, sd: SD, p: str, M: int) -> Tensor:
    """ExpandedFeatTrans without FFN, with the input skip: LN(coeff x + sum_m softmax_m(<w, y_m>) y_m), y_m = attn_m (x W_m^T)."""
    b, n, c = x.shape
    v = F.linear(x, sd[p + "first_linear.weight"]).view(b, n, M, -1).transpose(1, 2)  # [B, M, N, F]
    y = attn @ v
    pi = torch.softmax(F.linear(y, sd[p + "feat_softaggr.feat2score.weight"], sd[p + "feat_softaggr.feat2score.bias"]), dim=1)
    return ln(sd[p + "input_skip_coeff"] * x + (y * pi).sum(1))


def f2_transform(fmap2: Tensor, sd: SD, kw: dict) -> Tensor:
    b, c, h, w = fmap2.shape
    M = kw.get("f2_num_modes", 4)
    x = ln(tokens(fmap2))
    attn = probs(x, sd, "f2_trans.", M, kw.get("f2_pos_code_weight", 0.5), h, w, kw.get("f2_attn_mask_radius", -1))
    out = expanded(x, attn, sd, "f2_trans.setrans.out_trans.", M)
    return out.transpose(1, 2).reshape(b, c, h, w)


def mode_mix(s: Tensor, sd: SD, M: int) -> Tensor:
    """attn_softaggr of the scores [B, M, N, N] -> [B, N, N]: sum_m softmax_m(a s_m + b) s_m (one mode: s)."""
    if M == 1:
        return s[:, 0]
    p = "corr_fn.setrans.attn_softaggr.feat2score."
    pi = torch.softmax(sd[p + "weight"].reshape(()) * s + sd[p + "bias"].reshape(()), dim=1)
    return (pi * s).sum(1)


def craft_volume(fmap1: Tensor, fmap2t: Tensor, sd: SD, kw: dict, trace: Optional[dict] = None) -> Tensor:
    """[B*N, 1, H, W]."""
    b, c, h, w = fmap1.shape
    M = kw.get("inter_num_modes", 4)
    raw = mode_scores(ln(tokens(fmap1)), ln(tokens(fmap2t)), sd, "corr_fn.setrans.", M)
    s = clamp(raw) + kw.get("inter_pos_code_weight", 0.5) * window_bias(sd["corr_fn.vispos_encoder.pos_coder.biases"], h, w)
    mix = mode_mix(s, sd, M)
    if trace is not None:
        trace.update(raw_scores=raw, mix=mix)
    vol = F.layer_norm(mix.reshape(b, 1, -1), (h * w * h * w,), eps=1e-12)
    return vol.reshape(b * h * w, 1, h, w)


def forward(sd: SD, images: Tensor, kw: dict, flow_init: Optional[Tensor] = None, trace: Optional[dict] = None):
    x, pads = O.preprocess(images)
    b = x.shape[0]
    fm = O.encoder(torch.cat([x[:, 0], x[:, 1]], 0), sd, "fnet.", "instance", False)
    f1, f2 = fm[:b], fm[b:]
    cn = O.encoder(x[:, 0], sd, "cnet.", "batch", False)
    net, inp = torch.tanh(cn[:, :128]), torch.relu(cn[:, 128:])
    H, W = f1.shape[-2:]
    f2t = f2_transform(f2, sd, kw)
    vol = craft_volume(f1, f2t, sd, kw, trace) if kw.get("craft", True) else O.corr_volume(f1, f2t)
    pyr = O.corr_pyramid(vol, LEVELS)
    Mi = kw.get("intra_num_modes", 4)
    attn = probs(tokens(inp), sd, "att.", Mi, kw.get("intra_pos_code_weight", 1.0), H, W)
    if trace is not None:
        trace.update(f2t=f2t, volume=vol, attention=attn)
    radius = kw.get("corr_radius", 4)
    radius = 4 if radius == -1 else radius
    coords0 = O.coords_grid(b, H, W)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    mask = None
    for _ in range(kw.get("iters", 32)):
        corr = O.corr_lookup(pyr, coords1, radius)
        motion = O.motion_encoder_basic(coords1 - coords0, corr, sd)
        mg = expanded(tokens(motion), attn, sd, "update_block.aggregator.", Mi).transpose(1, 2).reshape(motion.shape)
        net = O.sep_conv_gru(net, torch.cat([inp, motion, mg], 1), sd)
        mask, delta = O.mask_head(net, sd), O.flow_head(net, sd)
        coords1 = coords1 + delta
    flows = O.unpad(O.convex_upsample(coords1 - coords0, mask), pads)
    return {"flows": flows[:, None], "flow_small": coords1 - coords0}


def e2e_inputs(recipe):
    kw = dict(recipe["kwargs"])
    return synth_state_dict(kw, recipe["wseed"], recipe.get("qscale", 1.0)), images(recipe), kw


def forward_recipe(recipe, flow_init: Optional[Tensor] = None, trace: Optional[dict] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(sd, img, kw, flow_init, trace)
