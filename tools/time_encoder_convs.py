#!/usr/bin/env python
"""The encoders' stride-1 3x3 convolutions of the bench workload (RAFT, 1024x436 padded to 440, 8 pairs, f16): cuDNN as
the encoders' planned convolutions (_EncConv in models/raft/extractor.py) call it against pfb_enc_conv3x3, in one process.

  1. one eager fnet + cnet pass per path under torch.profiler (CUDA activities): device time per kernel;
  2. every eligible layer shape timed with CUDA events, 50 launches per sample, the two paths alternating, with TFLOP/s,
     GB/s and share of the data-sheet peak computed from the shapes, and the per-step total (fnet sees 16 images, cnet 8);
  3. the eager per-class split of whole steps (one stream, no encoder fork) for both paths.
The card's name and power limit are read in the same run.

    python tools/time_encoder_convs.py [--out RESULT.json] [--launches 50] [--rounds 5]

The full result (every sample, the profiler's kernel table) goes to --out, by default time_encoder_convs.json in the
system's temporary directory; the summary is printed.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
from argparse import Namespace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import ptlflow_b200 as pb
from ptlflow_b200 import _lib, ops
from ptlflow_b200.models.raft import extractor

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35  # H100 SXM data sheet: dense f16 tensor, HBM3
KC_NAMES = ["volume", "pool", "lookup", "onthefly", "conv", "upsample", "misc", "enc_affine", "enc_stats", "enc_conv1", "flowconv",
            "gather", "depthwise", "dw_layernorm"]


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        info["nvidia_smi"] = q
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "time_encoder_convs.json"))
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev, dt = "cuda:0", torch.float16
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(1234)
    model = pb.get_model("raft", args=Namespace(model=Namespace(iters=12))).eval().to(dev).to(dt)
    B, H, W = 8, 436, 1024
    images = torch.rand(B, 2, 3, H, W, device=dev).to(dt)
    frames = torch.zeros(2 * B, 440, 1024, 4, device=dev, dtype=dt)
    frames[..., :3] = torch.rand(2 * B, 440, 1024, 3, device=dev).to(dt) * 2 - 1
    res = {"card": card(), "workload": "raft 1024x436 (440 padded), 8 pairs, f16"}

    def encoders():
        f = model.fnet.forward_pm(frames)
        c = model.cnet.forward_pm(frames[:B])
        return f, c

    # ---- 1. profiler: device time per kernel, one eager encoder pass per path ----
    from torch.profiler import ProfilerActivity, profile

    res["profile"] = {}
    with torch.no_grad():
        for native in (False, True):
            extractor._NATIVE_ENC_CONV = native
            for _ in range(3):
                encoders()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                encoders()
                torch.cuda.synchronize()
            rows = []
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                if t > 0:
                    rows.append((ev.key, ev.count, t))
            rows.sort(key=lambda r: -r[2])
            total = sum(r[2] for r in rows)
            res["profile"]["native" if native else "cudnn"] = {
                "total_us": round(total, 1), "kernels": [{"name": k[:120], "count": n, "us": round(t, 1)} for k, n, t in rows[:25]]}
            print(f"encoders ({'native' if native else 'cudnn'}): {total / 1e3:.3f} ms device time", flush=True)
            for k, n, t in rows[:12]:
                print(f"   {t:9.1f} us  x{n:3d}  {k[:110]}", flush=True)

    # ---- 2. per layer: CUDA events, the two paths alternating ----
    extractor._NATIVE_ENC_CONV = True
    fblocks = model.fnet._prepared(dt, torch.device(dev))[2]
    cblocks = model.cnet._prepared(dt, torch.device(dev))[2]
    # (name, images, grid, the second block's conv1 or conv2 step, kind, layers of this kind per encoder pass)
    specs = []
    for lname, (hh, ww), blk in (("layer1", (220, 512), 1), ("layer2", (110, 256), 3), ("layer3", (55, 128), 5)):
        n_conv1 = 2 if lname == "layer1" else 1  # conv1 of layer2's and layer3's first block is strided
        specs.append((lname, "fnet", 2 * B, (hh, ww), fblocks[blk].convs[0], "linear", n_conv1 + 2))
        specs.append((lname, "cnet", B, (hh, ww), cblocks[blk].convs[0], "bias_relu", n_conv1))
        specs.append((lname, "cnet", B, (hh, ww), cblocks[blk].convs[1], "bias_relu_residual", 2))
    layers = []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        for lname, enc, nb, (hh, ww), step, kind, per_pass in specs:
            routed = step.route == "enc_conv3x3"
            # a layer the plan leaves on cuDNN: packed here from the same storage-rounded weights
            packed = step.packed if routed else ops.PackedConv([ops.ConvWeights(step.weight.float())], dt, dev,
                                                               src_channels=[step.weight.shape[1]])
            bias = step.bias
            cin, cout = packed.Cin, packed.Cout
            x = (torch.randn(nb, hh, ww, cin, device=dev) * 0.5).relu().to(dt)
            r = (torch.randn(nb, hh, ww, cout, device=dev) * 0.5).relu().to(dt)

            def cudnn():
                if kind == "linear":
                    return extractor._conv_pm(x, step.weight, 1, 1)
                if kind == "bias_relu":
                    y = torch.cudnn_convolution_relu(x.permute(0, 3, 1, 2), step.weight, step.bias_storage, (1, 1), (1, 1), (1, 1), 1)
                    return y.permute(0, 2, 3, 1)
                y = extractor._conv_pm(x, step.weight, 1, 1)
                return ops.bias_act(y, step.bias, relu=True, residual=r, out=y)

            def native():
                if kind == "linear":
                    return ops.enc_conv3x3(x, packed)
                if kind == "bias_relu":
                    return ops.enc_conv3x3(x, packed, _lib.ENC_CONV_BIAS_RELU, bias=bias)
                return ops.enc_conv3x3(x, packed, _lib.ENC_CONV_BIAS_RELU_RESIDUAL, bias=bias, residual=r)

            diff = (cudnn().float() - native().float()).abs().max().item()
            t = {"cudnn": [], "native": []}
            for _ in range(2):
                cudnn(); native()
            for _ in range(a.rounds):
                for path, fn in (("cudnn", cudnn), ("native", native)):
                    torch.cuda.synchronize()
                    ev0.record()
                    for _ in range(a.launches):
                        fn()
                    ev1.record()
                    ev1.synchronize()
                    t[path].append(ev0.elapsed_time(ev1) * 1e3 / a.launches)
            flop = 2.0 * nb * hh * ww * cout * cin * 9
            nbytes = 2.0 * nb * hh * ww * (cin + cout + (cout if kind == "bias_relu_residual" else 0))
            row = {"layer": lname, "encoder": enc, "images": nb, "grid": [hh, ww], "cin": cin, "cout": cout, "epilogue": kind,
                   "per_pass": per_pass, "routed_to_enc_conv": routed, "max_abs_diff": diff}
            for path in ("cudnn", "native"):
                us = statistics.median(t[path])
                row[path] = {"us": round(us, 2), "tflops": round(flop / us * 1e-6, 1), "gbs": round(nbytes / us * 1e-3, 1),
                             "share_of_peak": round(max(flop / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_TBS * 1e12)) / (us * 1e-6), 3),
                             "samples_us": [round(v, 2) for v in t[path]]}
            layers.append(row)
            print(f"{lname} {enc} {kind:20s} {nb:2d}x{hh}x{ww} {cin}->{cout}: cudnn {row['cudnn']['us']:8.1f} us "
                  f"({row['cudnn']['tflops']:6.1f} TFLOP/s)  native {row['native']['us']:8.1f} us ({row['native']['tflops']:6.1f} TFLOP/s)"
                  f"  x{per_pass}/pass  max|diff| {diff:.3g}", flush=True)
    res["layers"] = layers
    for path in ("cudnn", "native"):
        res[f"{path}_stride1_ms_per_step"] = round(sum(l[path]["us"] * l["per_pass"] for l in layers) / 1e3, 3)
    res["dispatch_stride1_ms_per_step"] = round(
        sum(l["native" if l["routed_to_enc_conv"] else "cudnn"]["us"] * l["per_pass"] for l in layers) / 1e3, 3)
    print(f"stride-1 3x3 per step: cudnn {res['cudnn_stride1_ms_per_step']} ms, native {res['native_stride1_ms_per_step']} ms, "
          f"as dispatched {res['dispatch_stride1_ms_per_step']} ms", flush=True)

    # ---- 3. eager per-class split of whole steps (one stream, no fork) ----
    lib = _lib.load()
    res["eager_steps"] = {}
    with torch.no_grad():
        model.use_cuda_graph = False
        model.fork_encoders = model.fork_flow = False
        for native in (False, True, False, True):
            extractor._NATIVE_ENC_CONV = native
            model({"images": images})
            torch.cuda.synchronize()
            lib.pfb_profile_enable(1)
            ev0.record()
            for _ in range(a.steps):
                model({"images": images})
            ev1.record()
            ms_arr, n_arr = (C.c_double * 16)(), (C.c_ulonglong * 16)()
            _lib.check(lib.pfb_profile_collect(ms_arr, n_arr, 16), "profile_collect")
            lib.pfb_profile_enable(0)
            step = ev0.elapsed_time(ev1) / a.steps
            split = {KC_NAMES[k]: round(ms_arr[k] / a.steps, 3) for k in range(len(KC_NAMES)) if n_arr[k]}
            key = "native" if native else "cudnn"
            res["eager_steps"].setdefault(key, []).append({"ms_per_step": round(step, 3), "classes_ms_per_step": split})
            print(f"eager step ({key}): {step:.3f} ms; {split}", flush=True)
    extractor._NATIVE_ENC_CONV = True
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("card", "cudnn_stride1_ms_per_step", "native_stride1_ms_per_step",
                                          "dispatch_stride1_ms_per_step")}))


if __name__ == "__main__":
    main()
