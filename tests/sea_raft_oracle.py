"""SEA-RAFT on top of the oracle (TEST INFRASTRUCTURE, like oracle/): the ResNet-FPN encoders, the ConvNeXt block, the update block,
the eval forward and the state-dict shapes, plus the recipes of the fixtures tests/make_sea_raft_golden.py writes.

Written from the formulas of ptlflow/models/sea_raft/{extractor,layer,update,sea_raft}.py (not from their code) over the building
blocks of oracle/raft_oracle.py:
  ResNetFPN:  relu(bn1(conv1 7x7/2)) -> BasicBlocks y = relu(bn2(conv2(relu(bn1(conv1 x))))), x' = relu(down(x) + y) -> final_conv
  ConvNeXt:   y = LayerNorm_c(dwconv7(x)) * ln_w + ln_b  (un-fused: (y - mean) / sqrt(var + 1e-6));  h = gelu(y W1^T + b1)
              out = final(x + gamma * (h W2^T + b2))
  update:     x = [inp | motion(flow, corr)] (RAFT's motion encoder);  net = block_i([net | x]) for every block
  forward:    net | ctx = init_conv(cnet(cat[img1, img2]));  flow = flow_head(net)[:2];  iters x {lookup, update, flow += head};
              flows = convex_upsample(flow, 0.25 upsample_weight(net))
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import raft_oracle as O
from oracle import synth

Tensor = torch.Tensor
SD = Dict[str, Tensor]

BLOCKS = {"resnet18": (2, 2, 2), "resnet34": (3, 4, 6)}

# end-to-end fixtures: (name, registered model, model kwargs, batch, H, W, image kind, weight seed, image seed)
E2E_CASES = [
    ("e2e_sea_raft_default_ragged", "sea_raft", dict(), 2, 132, 164, "smooth", 51, 61),
    ("e2e_sea_raft_m", "sea_raft_m", dict(), 1, 128, 192, "smooth", 52, 62),
    ("e2e_sea_raft_iters12", "sea_raft", dict(iters=12), 1, 128, 160, "smooth", 53, 63),
    ("e2e_sea_raft_altcorr", "sea_raft", dict(alternate_corr=True), 1, 128, 192, "smooth", 54, 64),
    ("e2e_sea_raft_iters0", "sea_raft", dict(iters=0), 1, 128, 192, "noise", 55, 65),
    ("e2e_sea_raft_l3r3b3", "sea_raft", dict(corr_levels=3, corr_radius=3, num_blocks=3), 1, 128, 160, "smooth", 56, 66),
]
E2E = [c[0] for c in E2E_CASES]
PRETRAIN = {"sea_raft": "resnet18", "sea_raft_s": "resnet18", "sea_raft_m": "resnet34", "sea_raft_l": "resnet34"}

# operator fixture op_sea_raft.npz: one ConvNeXt block and one update iteration on two grids
OP_GRIDS = ((2, 8, 12), (1, 9, 16))
OP_SEED = 91
OP_SAMPLES = 4096


def op_sample(numel: int) -> np.ndarray:
    """The seeded subset of an operator output stored in op_sea_raft.npz."""
    return np.sort(np.random.default_rng(5).choice(numel, min(numel, OP_SAMPLES), replace=False))


def gelu(x: Tensor) -> Tensor:
    return 0.5 * x * (1.0 + torch.erf(x * 0.7071067811865476))


# --------------------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------------------
def _conv_shapes(s, name: str, cout: int, cin: int, k: int) -> None:
    s[name + ".weight"], s[name + ".bias"] = (cout, cin, k, k), (cout,)


def _bn_shapes(s, name: str, c: int) -> None:
    for t in ("weight", "bias", "running_mean", "running_var"):
        s[f"{name}.{t}"] = (c,)
    s[name + ".num_batches_tracked"] = ()


def _fpn_shapes(s, p: str, cin: int, cout: int, pretrain: str, initial_dim: int = 64, block_dims=(64, 128, 256)) -> None:
    _conv_shapes(s, p + "conv1", initial_dim, cin, 7)
    _bn_shapes(s, p + "bn1", initial_dim)
    inp = initial_dim
    for li, (dim, n) in enumerate(zip(block_dims, BLOCKS[pretrain]), start=1):
        for i in range(n):
            q, stride = f"{p}layer{li}.{i}.", (1 if li == 1 else 2) if i == 0 else 1
            _conv_shapes(s, q + "conv1", dim, inp, 3)
            _conv_shapes(s, q + "conv2", dim, dim, 3)
            _bn_shapes(s, q + "bn1", dim)
            _bn_shapes(s, q + "bn2", dim)
            if stride != 1 or inp != dim:  # bn3 and downsample.1 are one module under two names
                _bn_shapes(s, q + "bn3", dim)
                _conv_shapes(s, q + "downsample.0", dim, inp, 1)
                _bn_shapes(s, q + "downsample.1", dim)
            inp = dim
    _conv_shapes(s, p + "final_conv", cout, block_dims[2], 1)


def state_dict_shapes(pretrain: str = "resnet18", iters: int = 4, corr_levels: int = 4, corr_radius: int = 4,
                      num_blocks: int = 2) -> Dict[str, Tuple[int, ...]]:
    """The reference SEA-RAFT's state_dict names and shapes, in its order (sea_raft.py:94-133)."""
    s: Dict[str, Tuple[int, ...]] = {}
    _fpn_shapes(s, "cnet.", 6, 256, pretrain)
    _conv_shapes(s, "init_conv", 256, 256, 3)
    _conv_shapes(s, "upsample_weight.0", 256, 128, 3)
    _conv_shapes(s, "upsample_weight.2", 576, 256, 1)
    _conv_shapes(s, "flow_head.0", 256, 128, 3)
    _conv_shapes(s, "flow_head.2", 6, 256, 3)
    if iters > 0:
        _fpn_shapes(s, "fnet.", 3, 256, pretrain)
        e = "update_block.encoder."
        for name, cout, cin, k in (("convc1", 256, corr_levels * (2 * corr_radius + 1) ** 2, 1), ("convc2", 192, 256, 3),
                                   ("convf1", 128, 2, 7), ("convf2", 64, 128, 3), ("conv", 126, 256, 3)):
            _conv_shapes(s, e + name, cout, cin, k)
        for i in range(num_blocks):
            r = f"update_block.refine.{i}."
            s[r + "gamma"] = (384,)
            s[r + "dwconv.weight"], s[r + "dwconv.bias"] = (384, 1, 7, 7), (384,)
            s[r + "norm.weight"], s[r + "norm.bias"] = (384,), (384,)
            s[r + "pwconv1.weight"], s[r + "pwconv1.bias"] = (512, 384), (512,)
            s[r + "pwconv2.weight"], s[r + "pwconv2.bias"] = (384, 512), (384,)
            _conv_shapes(s, r + "final", 128, 384, 1)
    return s


def synth_state_dict(shapes, seed: int) -> SD:
    """oracle.synth weights, with every term of the ConvNeXt block made to show: the Linear layers N(0, 1/(3 fan_in)) like the
    convolutions (oracle.synth would give them a bias's 0.05), the LayerNorm weight 1 + 0.2 N and bias 0.2 N, and gamma
    0.5 + 0.1 N (O(1); the reference's 1e-6 initial value would hide the whole pwconv branch).  BatchNorm statistics are
    oracle.synth's (not the identity).  The encoders' convolutions get N(0, 1/fan_in) instead of kaiming's 2/fan_in: with eval
    BatchNorm nothing renormalises the residual stages, and at kaiming scale the 16 blocks of resnet34 grow the features (and the
    flow) by orders of magnitude."""
    sd = synth.synth_state_dict(shapes, seed)
    for k, shp in shapes.items():
        if len(shp) == 4 and k.startswith(("fnet.", "cnet.")):
            sd[k] = torch.from_numpy(synth.synth_normal(k, shp, seed, scale=float(np.prod(shp[1:])) ** -0.5))
        elif len(shp) == 2:
            sd[k] = torch.from_numpy(synth.synth_normal(k, shp, seed, scale=(3.0 * shp[1]) ** -0.5))
        elif k.endswith("norm.weight") and ".refine." in k:
            sd[k] = torch.from_numpy(1.0 + synth.synth_normal(k, shp, seed, scale=0.2))
        elif k.endswith("norm.bias") and ".refine." in k:
            sd[k] = torch.from_numpy(synth.synth_normal(k, shp, seed, scale=0.2))
    return sd


def e2e_inputs(recipe):
    """(state_dict, images, registered model name, kwargs) of an e2e_sea_raft_* fixture."""
    kw = dict(recipe["kwargs"])
    name = recipe["model"]
    shapes = state_dict_shapes(PRETRAIN[name], kw.get("iters", 12 if name == "sea_raft_l" else 4), kw.get("corr_levels", 4),
                               kw.get("corr_radius", 4), kw.get("num_blocks", 2))
    sd = synth_state_dict(shapes, recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, name, kw


def op_inputs(b: int, h: int, w: int):
    """(state dict, net, inp, corr, flow) of the op_sea_raft cases (default model, iters = 1)."""
    sd = synth_state_dict(state_dict_shapes(iters=1), OP_SEED)
    r = lambda name, shape, scale=1.0: torch.from_numpy(synth.synth_normal(name, shape, OP_SEED, scale=scale))  # noqa: E731
    net, inp = r("srop/net", (b, 128, h, w)), r("srop/inp", (b, 128, h, w))
    corr, flow = r("srop/corr", (b, 324, h, w)), r("srop/flow", (b, 2, h, w), 3.0)
    return sd, net, inp, corr, flow


# --------------------------------------------------------------------------------------
# blocks
# --------------------------------------------------------------------------------------
def resnet_fpn(x: Tensor, sd: SD, p: str, pretrain: str) -> Tensor:
    """ResNetFPN with eval-mode BatchNorm (extractor.py:105-116, layer.py:144-150)."""
    x = torch.relu(O._norm(O._conv(x, sd, p + "conv1", stride=2, padding=3), sd, p + "bn1", "batch"))
    for li, n in enumerate(BLOCKS[pretrain], start=1):
        for i in range(n):
            q, stride = f"{p}layer{li}.{i}.", (1 if li == 1 else 2) if i == 0 else 1
            y = torch.relu(O._norm(O._conv(x, sd, q + "conv1", stride=stride, padding=1), sd, q + "bn1", "batch"))
            y = torch.relu(O._norm(O._conv(y, sd, q + "conv2", padding=1), sd, q + "bn2", "batch"))
            if q + "downsample.0.weight" in sd:
                x = O._norm(O._conv(x, sd, q + "downsample.0", stride=stride), sd, q + "downsample.1", "batch")
            x = torch.relu(x + y)
    return O._conv(x, sd, p + "final_conv")


def convnext_block(x: Tensor, sd: SD, p: str) -> Tensor:
    """ConvNextBlock (layer.py:71-83) with the LayerNorm, GELU, gamma, residual and final written out separately."""
    c, k = x.shape[1], sd[p + "dwconv.weight"].shape[-1]
    y = F.conv2d(x, sd[p + "dwconv.weight"], sd[p + "dwconv.bias"], padding=k // 2, groups=c).permute(0, 2, 3, 1)
    mu = y.mean(-1, keepdim=True)
    var = ((y - mu) ** 2).mean(-1, keepdim=True)
    y = (y - mu) / torch.sqrt(var + 1e-6) * sd[p + "norm.weight"] + sd[p + "norm.bias"]
    h = gelu(y @ sd[p + "pwconv1.weight"].t() + sd[p + "pwconv1.bias"])
    y = sd[p + "gamma"] * (h @ sd[p + "pwconv2.weight"].t() + sd[p + "pwconv2.bias"])
    return O._conv(x + y.permute(0, 3, 1, 2), sd, p + "final")


def update_block(net: Tensor, inp: Tensor, corr: Tensor, flow: Tensor, sd: SD, num_blocks: int = 2) -> Tensor:
    """BasicUpdateBlock (update.py:49-54): RAFT's motion encoder, then the ConvNeXt blocks on [net | inp | motion]."""
    x = torch.cat([inp, O.motion_encoder_basic(flow, corr, sd)], 1)
    for i in range(num_blocks):
        net = convnext_block(torch.cat([net, x], 1), sd, f"update_block.refine.{i}.")
    return net


def flow_delta(net: Tensor, sd: SD) -> Tensor:
    """flow_head(net)[:, :2] (sea_raft.py:195, 225)."""
    return O._conv(torch.relu(O._conv(net, sd, "flow_head.0", padding=1)), sd, "flow_head.2", padding=1)[:, :2]


def upsample_mask(net: Tensor, sd: SD) -> Tensor:
    return 0.25 * O._conv(torch.relu(O._conv(net, sd, "upsample_weight.0", padding=1)), sd, "upsample_weight.2")


def iteration(net, inp, corr, flow, sd: SD, num_blocks: int = 2):
    """One update iteration -> (net, delta, mask)."""
    net = update_block(net, inp, corr, flow, sd, num_blocks)
    return net, flow_delta(net, sd), upsample_mask(net, sd)


def forward(sd: SD, images: Tensor, pretrain: str = "resnet18", iters: int = 4, corr_levels: int = 4, corr_radius: int = 4,
            num_blocks: int = 2, alternate_corr: bool = False, **_) -> Dict[str, Tensor]:
    """Eval-mode SEA-RAFT forward (sea_raft.py:165-276)."""
    sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
    x, pads = O.preprocess(images.float())
    img1, img2 = x[:, 0], x[:, 1]
    cnet = O._conv(resnet_fpn(torch.cat([img1, img2], 1), sd, "cnet.", pretrain), sd, "init_conv", padding=1)
    net, ctx = cnet[:, :128], cnet[:, 128:256]
    flow = flow_delta(net, sd)
    if iters > 0:
        b = img1.shape[0]
        fmaps = resnet_fpn(torch.cat([img1, img2], 0), sd, "fnet.", pretrain)
        fmap1, fmap2 = fmaps[:b], fmaps[b:]
        pyramid = None if alternate_corr else O.corr_pyramid(O.corr_volume(fmap1, fmap2), corr_levels)
        coords0 = O.coords_grid(b, *fmap1.shape[-2:], device=fmap1.device)
    for _ in range(iters):
        coords1 = coords0 + flow
        if alternate_corr:
            corr = O.alt_corr_lookup(fmap1, fmap2, coords1, corr_radius, corr_levels)
        else:
            corr = O.corr_lookup(pyramid, coords1, corr_radius)
        net = update_block(net, ctx, corr, flow, sd, num_blocks)
        flow = flow + flow_delta(net, sd)
    flows = O.unpad(O.convex_upsample(flow, upsample_mask(net, sd)), pads)
    return {"flows": flows[:, None], "flow_small": flow}


def forward_recipe(recipe) -> Dict[str, Tensor]:
    sd, img, name, kw = e2e_inputs(recipe)
    kw = dict(kw)
    kw.setdefault("iters", 12 if name == "sea_raft_l" else 4)
    return forward(sd, img, PRETRAIN[name], **kw)
