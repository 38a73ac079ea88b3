"""CCMR / CCMR+ on top of tests/ms_raft_oracle.py (TEST INFRASTRUCTURE, like oracle/): the XCiT block written from its definition,
the encoders' after-up 1x1 convolutions, the scale loop with the flow handover, upflow2, and the recipes of the fixtures
tests/make_ccmr_golden.py writes.

Written from the formulas of ptlflow/models/ccmr/{xcit,extractor,update,ccmr,utils}.py, fp32 on the CPU:
  pos:       64 Fourier features of the normalised cumulative row / column index (sin, cos interleaved), then token_projection
  XCA:       q, k, v = 16-channel heads of the linears of LN1;  q^, k^ = q, k / max(||.||_N, 1e-12) over the N pixels;
             A_h = softmax_j(t_h q^_i . k^_j);  out = proj(A_h v)   (the aggregator: q, k from LN1(gc + pos), v from LN1(motion))
  block:     x += g1 XCA;  x += g3 LPI(LN3 x), LPI = dw3x3 -> GELU -> GroupNorm(8) -> dw3x3;  x += g2 fc2(GELU(fc1(LN2 x)))
  scale i:   gc = XCiT_i(inp);  iterations of the update block with GRU input [inp | motion | aggregator_i(gc, motion)];  at the start
             of scale i >= 1, coords = grid_i + convex2x(coords - grid_{i-1}, previous mask)
  output:    flows = convex2x(coords - grid) of the last scale, then (ccmr) upflow2, un-padded;  flow_small = downflow(flows, 1/16)
The XCA is formed explicitly here (normalisation, gram, softmax, A v), so the device's fold is tested against it, not restated.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

import ms_raft_oracle as MS
from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]

# end-to-end fixtures: (name, model, model kwargs, batch, H, W, image kind, weight seed, image seed, warm start)
E2E_CASES = [
    ("e2e_ccmr_default", "ccmr", dict(), 1, 64, 96, "smooth", 171, 181, False),
    ("e2e_ccmr_p_default", "ccmr_p", dict(), 1, 64, 96, "smooth", 172, 182, False),
    ("e2e_ccmr_p_ragged_b2", "ccmr_p", dict(iters=(2, 2, 1, 2)), 2, 72, 104, "smooth", 173, 183, False),
    ("e2e_ccmr_warm", "ccmr", dict(iters=(2, 3, 2)), 1, 64, 96, "smooth", 174, 184, True),
    ("e2e_ccmr_p_volume", "ccmr_p", dict(alternate_corr=False, iters=(2, 2, 2, 2)), 1, 64, 64, "smooth", 175, 185, False),
]
E2E = [c[0] for c in E2E_CASES]
OP_SEED = 193
NUM_SCALES = {"ccmr": 3, "ccmr_p": 4}
DEFAULT_ITERS = {"ccmr": (8, 10, 15), "ccmr_p": (8, 10, 10, 10)}


def recipe_of(case) -> dict:
    name, model, kw, b, h, w, kind, ws, iseed, warm = case
    return dict(model=model, kwargs=kw, batch=b, height=h, width=w, kind=kind, wseed=ws, iseed=iseed, warm=warm)


def synth_state_dict(shapes, seed: int) -> SD:
    """oracle.synth weights, with every XCiT term of order 1: gamma1/2/3 = 1 + 0.1 N (the reference initialises eta = 1),
    temperature = 1 + 0.3 N per head, the XCiT linears at unit gain (N(0, 1/fan_in)) and non-identity LayerNorm / GroupNorm
    affines (1 + 0.1 N, 0.05 N)."""
    sd = synth.synth_state_dict(shapes, seed)
    for k, shape in shapes.items():
        g = synth._gen(seed, "ccmr/" + k)
        if ".gamma" in k.rsplit(".", 1)[-1] or k.endswith(("gamma1", "gamma2", "gamma3")):
            sd[k] = torch.from_numpy((1.0 + 0.1 * g.standard_normal(shape)).astype("float32"))
        elif k.endswith("temperature"):
            sd[k] = torch.from_numpy((1.0 + 0.3 * g.standard_normal(shape)).astype("float32"))
        elif ("xcit." in k or "aggregator." in k) and k.endswith("weight") and len(shape) == 2:
            sd[k] = torch.from_numpy((g.standard_normal(shape) / math.sqrt(shape[1])).astype("float32"))
    return sd


# --------------------------------------------------------------------------------------
# XCiT
# --------------------------------------------------------------------------------------
def _ln(x: Tensor, sd: SD, name: str) -> Tensor:  # x [B, N, C]
    return F.layer_norm(x, x.shape[-1:], sd[name + ".weight"], sd[name + ".bias"], eps=1e-6)


def _lin(x: Tensor, sd: SD, name: str) -> Tensor:
    return F.linear(x, sd[name + ".weight"], sd.get(name + ".bias"))


def fourier_pos(sd: SD, p: str, B: int, H: int, W: int) -> Tensor:
    """PositionalEncodingFourier(hidden_dim=32, dim=128) -> [B, N, 128]."""
    y = torch.arange(1, H + 1, dtype=torch.float32)[:, None].expand(H, W)
    x = torch.arange(1, W + 1, dtype=torch.float32)[None, :].expand(H, W)
    y = y / (H + 1e-6) * (2 * math.pi)
    x = x / (W + 1e-6) * (2 * math.pi)
    d = torch.arange(32, dtype=torch.float32)
    dim_t = 10000 ** (2 * (d // 2) / 32)

    def enc(e):
        a = e[..., None] / dim_t
        return torch.where((torch.arange(32) % 2 == 0), torch.sin(a), torch.cos(a))

    feat = torch.cat([enc(y), enc(x)], -1).reshape(1, H * W, 64)
    w = sd[p + "pos_embeder.token_projection.weight"][:, :, 0, 0]
    return (feat @ w.t() + sd[p + "pos_embeder.token_projection.bias"]).expand(B, -1, -1)


def xca(q: Tensor, k: Tensor, v: Tensor, temperature: Tensor, heads: int = 8) -> Tensor:
    """q, k, v [B, N, C] -> [B, N, C]: per head, L2-normalise q and k over N, A = softmax(t q^ k^T) (dh x dh), out = A v."""
    B, N, C = q.shape
    d = C // heads
    sp = lambda t: t.reshape(B, N, heads, d).permute(0, 2, 3, 1)  # noqa: E731  [B, h, d, N]
    qh, kh, vh = sp(q), sp(k), sp(v)
    qh = qh / qh.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    kh = kh / kh.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    a = torch.softmax((qh @ kh.transpose(-2, -1)) * temperature.reshape(1, heads, 1, 1), dim=-1)
    return (a @ vh).permute(0, 3, 1, 2).reshape(B, N, C)


def lpi(x: Tensor, sd: SD, p: str, H: int, W: int) -> Tensor:
    B, N, C = x.shape
    t = x.transpose(1, 2).reshape(B, C, H, W)
    t = F.conv2d(t, sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1, groups=C)
    t = F.group_norm(F.gelu(t), 8, sd[p + "bn.weight"], sd[p + "bn.bias"], eps=1e-5)
    t = F.conv2d(t, sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1, groups=C)
    return t.reshape(B, C, N).transpose(1, 2)


def xcit(sd: SD, p: str, x: Tensor, x_v: Optional[Tensor] = None) -> Tensor:
    """XCiT(depth=1) of xcit.py:406-427: x (and x_v for the aggregator) [B, C, H, W] -> [B, C, H, W]."""
    B, C, H, W = x.shape
    t = x.flatten(2).transpose(1, 2) + fourier_pos(sd, p, B, H, W)
    b = p + "blocks.0."
    n1 = _ln(t, sd, b + "norm1")
    if x_v is None:
        qkv = _lin(n1, sd, b + "attn.qkv")
        q, k, v = qkv[..., :C], qkv[..., C : 2 * C], qkv[..., 2 * C :]
    else:
        qk = _lin(n1, sd, b + "attn.to_qk")
        q, k = qk[..., :C], qk[..., C:]
        v = _lin(_ln(x_v.flatten(2).transpose(1, 2), sd, b + "norm1"), sd, b + "attn.to_v")
    t = t + sd[b + "gamma1"] * _lin(xca(q, k, v, sd[b + "attn.temperature"]), sd, b + "attn.proj")
    t = t + sd[b + "gamma3"] * lpi(_ln(t, sd, b + "norm3"), sd, b + "local_mp.", H, W)
    t = t + sd[b + "gamma2"] * _lin(F.gelu(_lin(_ln(t, sd, b + "norm2"), sd, b + "mlp.fc1")), sd, b + "mlp.fc2")
    return t.transpose(1, 2).reshape(B, C, H, W)


# --------------------------------------------------------------------------------------
# encoders, update block, loop
# --------------------------------------------------------------------------------------
def pyramid_encoder(x: Tensor, sd: SD, p: str, scales: int):
    x = torch.relu(MS.group_norm(O._conv(x, sd, p + "conv1", stride=2, padding=3), sd, p + "norm1"))
    e1 = MS.layer(x, sd, p + "layer1", 1)
    e2 = MS.layer(e1, sd, p + "layer2", 2)
    e3 = MS.layer(e2, sd, p + "layer3", 2)
    outs = [O._conv(MS.layer(e3, sd, p + "layer4", 2), sd, p + "conv2")]
    for k, skip in zip(range(2, 2 - (scales - 1), -1), (e3, e2, e1)):
        u = MS.up_layer(outs[-1], skip, sd, f"{p}up_layer{k}")
        outs.append(O._conv(u, sd, f"{p}after_up_layer{k}_conv"))
    return outs


def upflow2(flow: Tensor) -> Tensor:
    return 2 * F.interpolate(flow, scale_factor=2, mode="bilinear", align_corners=True)


def update_block(net, inp, corr, flow, gc, sd: SD, i: int):
    """-> (net, mask [B,36,H,W] (x0.25), delta): ccmr/update.py:156-168."""
    motion = O.motion_encoder_basic(flow, corr, sd)
    glob = xcit(sd, f"update_block.aggregator.{i}.", gc, motion)
    net = O.sep_conv_gru(net, torch.cat([inp, motion, glob], 1), sd)
    mask, delta = O.mask_head(net, sd), O.flow_head(net, sd)
    return net, mask, delta


def forward(sd: SD, images: Tensor, model: str = "ccmr", iters=None, levels: int = 2, radius: int = 4, alternate_corr: bool = True,
            flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    S = NUM_SCALES[model]
    iters = DEFAULT_ITERS[model] if iters is None else iters
    x = torch.flip((images + (-0.5)) * 2.0, dims=[-3])
    pads = O.pad_amounts(x.shape[-2], x.shape[-1], 32)
    b = x.shape[0]
    x = F.pad(x.reshape(2 * b, *x.shape[2:]), pads, mode="replicate").reshape(b, 2, 3, x.shape[-2] + pads[2] + pads[3], -1)
    fp = pyramid_encoder(torch.cat([x[:, 0], x[:, 1]], 0), sd, "fnet.", S)
    cp = pyramid_encoder(x[:, 0], sd, "cnet.", S)
    H, W = fp[0].shape[-2:]
    coords0 = O.coords_grid(b, H, W)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init
    mask = None
    for i in range(S):
        f1, f2 = fp[i][:b], fp[i][b:]
        if alternate_corr:
            lookup = lambda c: O.alt_corr_lookup(f1, f2, c, radius, levels)  # noqa: E731
        else:
            pyr = O.corr_pyramid(O.corr_volume(f1, f2), levels)
            lookup = lambda c: O.corr_lookup(pyr, c, radius)  # noqa: E731
        net, inp = torch.tanh(cp[i][:, :128]), torch.relu(cp[i][:, 128:])
        gc = xcit(sd, f"xcit.{i}.", inp)
        if i > 0:
            flow = MS.convex_up2(coords1 - coords0, mask)
            coords0 = O.coords_grid(b, *flow.shape[-2:])
            coords1 = coords0 + flow
        for _ in range(iters[i]):
            net, mask, delta = update_block(net, inp, lookup(coords1), coords1 - coords0, gc, sd, i)
            coords1 = coords1 + delta
    flows = MS.convex_up2(coords1 - coords0, mask)
    for _ in range((S - 1 if S == 4 else S) - (S - 1)):
        flows = upflow2(flows)
    flows = O.unpad(flows, pads)
    return {"flows": flows[:, None], "flow_small": MS.downflow(flows)}


def state_dict_shapes(model: str):
    """The reference's state_dict names and shapes, as written by tests/make_ccmr_golden.py."""
    import json
    import os

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"state_shapes_{model}.json")) as f:
        return {k: tuple(v) for k, v in json.load(f).items()}


def e2e_inputs(recipe):
    kw = dict(recipe["kwargs"])
    sd = synth_state_dict(state_dict_shapes(recipe["model"]), recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


def forward_recipe(recipe, flow_init: Optional[Tensor] = None) -> Dict[str, Tensor]:
    sd, img, kw = e2e_inputs(recipe)
    with O.fp32_strict(), torch.no_grad():
        return forward(sd, img, recipe["model"], kw.get("iters"), 2, 4, kw.get("alternate_corr", True), flow_init)


def op_inputs():
    """Inputs of op_ccmr.npz (the ccmr_p weights): a context map for XCiT, one update iteration's (net, inp, corr, flow, gc) at
    scale 1, a (coords, mask) pair for the scale handover and a flow for upflow2."""
    sd = synth_state_dict(state_dict_shapes("ccmr_p"), OP_SEED)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    x = {
        "ctx": torch.relu(r("ccmrop/ctx", (2, 128, 6, 9))),
        "net": torch.tanh(r("ccmrop/net", (2, 128, 6, 9))),
        "inp": torch.relu(r("ccmrop/inp", (2, 128, 6, 9))),
        "corr": r("ccmrop/corr", (2, 162, 6, 9)),
        "flow": r("ccmrop/flow", (2, 2, 6, 9), 3.0),
        "mask": r("ccmrop/mask", (2, 36, 6, 9), 2.0),
        "flow_lo": r("ccmrop/flow_lo", (2, 2, 5, 7), 3.0),
    }
    x["gc"] = r("ccmrop/gc", (2, 128, 6, 9))
    x["coords"] = O.coords_grid(2, 6, 9) + r("ccmrop/coords", (2, 2, 6, 9), 4.0)
    return sd, x


np32 = MS.np32
