"""Time SKFlow at the BASELINE config-3 image size (1024x436, 12 iterations).

    python tools/time_skflow.py [--steps 20] [--warmup 5] [--reps 50]

1. The model: ``skflow`` with default hparams (random-init weights, seed 1234, torch.rand frames), bf16 and f16, batch 4 and 8,
   one CUDA graph launch per forward.  Pairs/s from CUDA events around --steps forwards after --warmup forwards (the first ones
   capture the graph).
2. The per-kernel-class split of one eager forward (pfb_profile_enable / pfb_profile_collect; class 12 = depthwise).
3. The depthwise kernel alone for each depthwise layer of the default update block at the batch-8 grid (55x128): time from CUDA
   events around --reps launches, FLOP = 2 k^2 C per pixel, and the share of the H100 SXM's 67 TFLOP/s fp32 (non-tensor) peak.

Prints one JSON line per measurement, each with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
from argparse import Namespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KC_NAMES = ["volume", "pool", "lookup", "onthefly", "conv", "upsample", "misc", "enc_affine", "enc_stats", "enc_conv1", "flowconv",
            "gather", "depthwise"]
FP32_PEAK = 67e12
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({type(e).__name__})"}


def events_ms(fn, n: int) -> float:
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / n


def time_model(args, dname, batch, info) -> None:
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib

    dtype = DTYPES[dname]
    torch.manual_seed(1234)
    model = pb.get_model("skflow", args=Namespace(model=Namespace(iters=args.iters))).eval().cuda().to(dtype)
    frames = [torch.rand(batch, 2, 3, args.height, args.width, device="cuda").to(dtype) for _ in range(3)]
    step = [0]

    def fwd():
        model({"images": frames[step[0] % 3]})
        step[0] += 1

    with torch.no_grad():
        for _ in range(args.warmup):
            fwd()
        torch.cuda.synchronize()
        ms = events_ms(fwd, args.steps)
        # per-kernel-class split of one eager forward
        lib = _lib.load()
        model.use_cuda_graph = False
        fwd()
        torch.cuda.synchronize()
        lib.pfb_profile_enable(1)
        fwd()
        ms_arr, n_arr = (C.c_double * 16)(), (C.c_ulonglong * 16)()
        _lib.check(lib.pfb_profile_collect(ms_arr, n_arr, 16), "profile_collect")
        lib.pfb_profile_enable(0)
    split = {KC_NAMES[i]: {"ms": round(ms_arr[i], 3), "launches": int(n_arr[i])} for i in range(len(KC_NAMES)) if n_arr[i]}
    print(json.dumps({"model": "skflow", "dtype": dname, "batch": batch, "image": [args.height, args.width], "iters": args.iters,
                      "ms_per_step": round(ms, 3), "pairs_per_s": round(batch / (ms * 1e-3), 1), "steps": args.steps,
                      "eager_kernel_split": split, **info}), flush=True)
    del model, frames
    torch.cuda.empty_cache()


def time_depthwise(args, dname, batch, info) -> None:
    from ptlflow_b200 import ops

    dtype = DTYPES[dname]
    H, W = -(-args.height // 8), -(-args.width // 8)
    P = batch * H * W
    # (layer, padded channels, k) of the default model's depthwise steps (the k = 1 entries ride the ffn1 epilogue)
    layers = [("encoder.convc1", 352, 15), ("encoder.convc2", 256, 15), ("encoder.convf2", 128, 15), ("encoder.conv", 256, 15),
              ("gru", 512, 7), ("flow_head", 128, 15)]
    total_ms = total_flop = 0.0
    for name, Cc, k in layers:
        x = torch.randn(batch, H, W, Cc, device="cuda").to(dtype)
        out = torch.empty_like(x)
        w, b = torch.randn(k * k, Cc, device="cuda") / k, torch.randn(Cc, device="cuda")
        for _ in range(3):
            ops.depthwise_conv_gelu(x, w, b, k, out=out)
        ms = events_ms(lambda: ops.depthwise_conv_gelu(x, w, b, k, out=out), args.reps)
        flop = 2.0 * k * k * Cc * P
        total_ms, total_flop = total_ms + ms, total_flop + flop
        print(json.dumps({"kernel": "pfb_depthwise_conv_gelu", "layer": name, "C": Cc, "k": k, "batch": batch, "grid": [H, W], "dtype": dname,
                          "ms": round(ms, 4), "TFLOP_per_s": round(flop / (ms * 1e-3) / 1e12, 2),
                          "fp32_peak_fraction_vs_67TF": round(flop / (ms * 1e-3) / FP32_PEAK, 3), **info}), flush=True)
        del x, out
    print(json.dumps({"kernel": "pfb_depthwise_conv_gelu", "layer": "all per iteration", "batch": batch, "dtype": dname,
                      "ms": round(total_ms, 4), "GFLOP": round(total_flop / 1e9, 2), "TFLOP_per_s": round(total_flop / (total_ms * 1e-3) / 1e12, 2),
                      "fp32_peak_fraction_vs_67TF": round(total_flop / (total_ms * 1e-3) / FP32_PEAK, 3), **info}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=436)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=12)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    info = card()
    for dname in ("bf16", "fp16"):
        for batch in (4, 8):
            time_model(args, dname, batch, info)
    time_depthwise(args, "bf16", 8, info)


if __name__ == "__main__":
    main()
