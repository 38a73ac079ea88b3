#!/usr/bin/env python
"""Where does the half-precision error of the flow come from?  (CPU tool, TEST INFRASTRUCTURE.)

Re-runs the oracle's RAFT forward (oracle/raft_oracle.py, fp32 arithmetic) with the *storage
roundings* of the CUDA pipeline injected at the places where the kernels round to f16 / bf16:
weights, frames, encoder activations, feature maps, the correlation pyramid, the lookup output,
the motion-encoder / GRU / head activations and the hidden state.  Every group can be switched
on alone ("only") or off alone ("all but"), which gives the error budget of the half path against
the fp32 reference without a GPU (accumulation is fp32 in both, as in the kernels).

    python tools/f16_error_budget.py [--dtype f16|bf16] [--case e2e_raft_noise ...]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from oracle import raft_oracle as O  # noqa: E402

GROUPS = ["w_enc", "w_upd", "img", "enc_raw", "enc_act", "fmap", "ctx", "vol", "lookup", "mot", "gate", "net", "head"]


class Rounder:
    def __init__(self, dtype, on):
        self.dtype, self.on = dtype, set(on)

    def __call__(self, group, x):
        if group in self.on:
            return x.to(self.dtype).float()
        return x


def forward(sd, images, rnd: Rounder, variant="raft", iters=12, alternate_corr=False, corr_levels=4, corr_radius=None):
    small, hdim, cdim, _f, cnorm, r_default = O.VARIANTS[variant]
    assert not small
    radius = r_default if corr_radius is None else corr_radius
    sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
    # weights as stored by the kernels: f16 weights, fp32 biases; batch norm folded in fp32 first (extractor._EncConv)
    sdw = {}
    for k, v in sd.items():
        if v.dim() == 4:
            sdw[k] = rnd("w_enc" if k.startswith(("fnet.", "cnet.")) else "w_upd", v)
        else:
            sdw[k] = v

    x, pads = O.preprocess(images.float())
    x = rnd("img", x)
    img1, img2 = x[:, 0], x[:, 1]
    b = img1.shape[0]

    def enc(xin, prefix, kind):
        def conv_norm(xx, name, normname, stride, padding, relu=True):
            w = sd[name + ".weight"]
            bias = sd.get(name + ".bias")
            if kind == "batch":
                s = sd[normname + ".weight"] / torch.sqrt(sd[normname + ".running_var"] + 1e-5)
                t = sd[normname + ".bias"] - sd[normname + ".running_mean"] * s
                w = w * s.view(-1, 1, 1, 1)
                bias = bias * s + t
            w = rnd("w_enc", w)
            y = F.conv2d(xx, w, None, stride=stride, padding=padding)
            y = rnd("enc_raw", y)  # cuDNN writes the raw convolution in the storage type
            if kind == "instance":
                y = F.instance_norm(y, eps=1e-5)
            else:
                y = y + bias.view(1, -1, 1, 1)
            return torch.relu(y) if relu else y

        y = rnd("enc_act", conv_norm(xin, prefix + "conv1", prefix + "norm1", 2, 3))
        for li, stride in ((1, 1), (2, 2), (3, 2)):
            for bi, st in ((0, stride), (1, 1)):
                p = f"{prefix}layer{li}.{bi}."
                xs = y
                if st != 1:
                    xs = rnd("enc_act", conv_norm(y, p + "downsample.0", p + "downsample.1", st, 0, relu=False))
                t = rnd("enc_act", conv_norm(y, p + "conv1", p + "norm1", st, 1))
                t = conv_norm(t, p + "conv2", p + "norm2", 1, 1)
                y = rnd("enc_act", torch.relu(xs + t))
        w = rnd("w_enc", sd[prefix + "conv2.weight"])
        y = rnd("enc_raw", F.conv2d(y, w, None)) + sd[prefix + "conv2.bias"].view(1, -1, 1, 1)
        return y

    fmaps = rnd("fmap", enc(torch.cat([img1, img2], 0), "fnet.", "instance"))
    fmap1, fmap2 = fmaps[:b], fmaps[b:]
    cnet = rnd("fmap", enc(img1, "cnet.", cnorm))
    net = rnd("ctx", torch.tanh(cnet[:, :hdim]))
    inp = rnd("ctx", torch.relu(cnet[:, hdim:hdim + cdim]))

    pyr = [rnd("vol", O.corr_volume(fmap1, fmap2))]
    for _ in range(corr_levels - 1):
        pyr.append(rnd("vol", O.corr_pyramid(pyr[-1], 2)[1]))
    h8, w8 = fmap1.shape[-2:]
    coords0 = O.coords_grid(b, h8, w8)
    coords1 = coords0.clone()

    def conv(xx, name, padding=0):
        return F.conv2d(xx, sdw[name + ".weight"], sdw.get(name + ".bias"), padding=padding)

    e, g = "update_block.encoder.", "update_block.gru."
    mask = None
    for it in range(iters):
        corr = rnd("lookup", O.corr_lookup(pyr, coords1, radius))
        flow = coords1 - coords0
        cor = rnd("mot", torch.relu(conv(corr, e + "convc1")))
        cor = rnd("mot", torch.relu(conv(cor, e + "convc2", 1)))
        flo = rnd("mot", torch.relu(conv(flow, e + "convf1", 3)))  # hi/lo split flow: exact fp32 flow x f16 weights
        flo = rnd("mot", torch.relu(conv(flo, e + "convf2", 1)))
        out = rnd("mot", torch.relu(conv(torch.cat([cor, flo], 1), e + "conv", 1)))
        motion = torch.cat([out, rnd("mot", flow)], 1)
        xcat = torch.cat([inp, motion], 1)
        for sfx, pad in (("1", (0, 2)), ("2", (2, 0))):
            hx = torch.cat([net, xcat], 1)
            z = rnd("gate", torch.sigmoid(conv(hx, g + "convz" + sfx, pad)))
            r = torch.sigmoid(conv(hx, g + "convr" + sfx, pad))
            rh = rnd("gate", r * net)
            q = torch.tanh(conv(torch.cat([rh, xcat], 1), g + "convq" + sfx, pad))
            net = rnd("net", (1 - z) * net + z * q)
        fh = rnd("head", torch.relu(conv(net, "update_block.flow_head.conv1", 1)))
        delta = conv(fh, "update_block.flow_head.conv2", 1)
        coords1 = coords1 + delta
        if it == iters - 1:
            mh = rnd("head", torch.relu(conv(net, "update_block.mask.0", 1)))
            mask = rnd("head", 0.25 * conv(mh, "update_block.mask.2"))
    flow_small = coords1 - coords0
    up = O.convex_upsample(flow_small, mask)
    return O.unpad(up, pads)[:, None]


def main():
    from helpers import e2e_inputs, load_golden

    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="f16")
    ap.add_argument("--case", nargs="*", default=["e2e_raft_noise", "e2e_raft_smooth_b2"])
    ap.add_argument("--threads", type=int, default=8)
    args = ap.parse_args()
    torch.set_num_threads(args.threads)
    dt = torch.float16 if args.dtype == "f16" else torch.bfloat16
    for case in args.case:
        recipe, gold = load_golden(case)
        sd, img, kw = e2e_inputs(recipe)
        iters = kw.get("iters", 12)
        with torch.no_grad():
            ref = forward(sd, img, Rounder(dt, []), recipe["variant"], iters)
            gerr = (ref.numpy() - gold["flows"]).__abs__().max()
            print(f"== {case}: {recipe['height']}x{recipe['width']} b{recipe['batch']} iters {iters}; no-rounding vs golden {gerr:.2e}")
            full = forward(sd, img, Rounder(dt, GROUPS), recipe["variant"], iters)
            d = (full - ref).abs()
            print(f"   all roundings on   : max {d.max():.4f}  mean {d.mean():.5f}")
            rows = []
            for grp in GROUPS:
                only = (forward(sd, img, Rounder(dt, [grp]), recipe["variant"], iters) - ref).abs()
                but = (forward(sd, img, Rounder(dt, [x for x in GROUPS if x != grp]), recipe["variant"], iters) - ref).abs()
                rows.append((grp, only.max().item(), only.mean().item(), but.max().item(), but.mean().item()))
                print(f"   {grp:8s} only: max {rows[-1][1]:.4f} mean {rows[-1][2]:.5f} | all but: max {rows[-1][3]:.4f} mean {rows[-1][4]:.5f}", flush=True)
            print(json.dumps({"case": case, "dtype": args.dtype, "all": [d.max().item(), d.mean().item()], "groups": rows}))


if __name__ == "__main__":
    main()
