"""Time SEA-RAFT at the BASELINE config-3 image size (1024x436).

    python tools/time_sea_raft.py [--steps 20] [--warmup 5] [--reps 50]

1. The models ``sea_raft_s`` (resnet18, 4 iterations) and ``sea_raft_l`` (resnet34, 12 iterations) with default hparams (random-init
   weights, seed 1234, torch.rand frames), f16 and bf16, batch 4 and 8, one CUDA graph launch per forward.  Pairs/s from CUDA
   events around --steps forwards after --warmup forwards (the first ones capture the graph).
2. One eager forward split by kernel class (pfb_profile_enable / pfb_profile_collect): encoders (this library's encoder passes),
   volume (build + pooling), loop convolutions (wgmma / SIMT convolutions, convf1, flow-head gather), depthwise + LayerNorm
   (class 13), and other = the eager forward's event time minus those (cuDNN's encoder convolutions, lookup, upsample, copies,
   launch gaps).
3. pfb_depthwise_conv_layernorm alone at the config-3 grid (55x128, C = 384, k = 7) for batch 4 and 8: time from CUDA events around
   --reps launches; bytes = one read of the input and one write of the output (the ideal), FLOP = 2 k^2 C per pixel; the share of
   the H100 SXM's 3.35 TB/s HBM bandwidth and of its 67 TFLOP/s fp32 (non-tensor) peak.

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
            "gather", "depthwise", "dw_layernorm"]
GROUPS = {"encoders": ("enc_affine", "enc_stats", "enc_conv1"), "volume": ("volume", "pool"), "loop_conv": ("conv", "flowconv", "gather"),
          "dw_layernorm": ("dw_layernorm",)}
FP32_PEAK, HBM_BW = 67e12, 3.35e12
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


def time_model(args, name, dname, batch, info) -> None:
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib

    dtype = DTYPES[dname]
    torch.manual_seed(1234)
    model = pb.get_model(name).eval().cuda().to(dtype)
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
        lib = _lib.load()
        model.use_cuda_graph = False
        fwd()
        torch.cuda.synchronize()
        eager_ms = events_ms(fwd, 1)
        lib.pfb_profile_enable(1)
        fwd()
        ms_arr, n_arr = (C.c_double * 16)(), (C.c_ulonglong * 16)()
        _lib.check(lib.pfb_profile_collect(ms_arr, n_arr, 16), "profile_collect")
        lib.pfb_profile_enable(0)
    per = {KC_NAMES[i]: ms_arr[i] for i in range(len(KC_NAMES))}
    split = {g: round(sum(per[k] for k in ks), 3) for g, ks in GROUPS.items()}
    split["other"] = round(eager_ms - sum(split.values()), 3)
    print(json.dumps({"model": name, "dtype": dname, "batch": batch, "image": [args.height, args.width], "iters": model.iters,
                      "ms_per_step": round(ms, 3), "pairs_per_s": round(batch / (ms * 1e-3), 1), "steps": args.steps,
                      "eager_forward_ms": round(eager_ms, 3), "eager_split_ms": split, **info}), flush=True)
    del model, frames
    torch.cuda.empty_cache()


def time_kernel(args, dname, batch, info) -> None:
    from ptlflow_b200 import ops

    dtype = DTYPES[dname]
    H, W, Cc, k = (args.height + 7) // 8, (args.width + 7) // 8, 384, 7
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(batch, H, W, Cc, device="cuda", generator=g).to(dtype)
    w = torch.randn(k * k, Cc, device="cuda", generator=g) / k
    b = torch.randn(Cc, device="cuda", generator=g) * 0.1
    out = torch.empty_like(x)
    for _ in range(5):
        ops.depthwise_conv_layernorm(x, w, b, k, out=out)
    ms = events_ms(lambda: ops.depthwise_conv_layernorm(x, w, b, k, out=out), args.reps)
    P = batch * H * W
    nbytes = 2 * P * Cc * x.element_size()
    flop = 2 * k * k * Cc * P
    t = ms * 1e-3
    print(json.dumps({"kernel": "pfb_depthwise_conv_layernorm", "C": Cc, "k": k, "batch": batch, "grid": [H, W], "dtype": dname,
                      "us": round(ms * 1e3, 2), "GB_per_s": round(nbytes / t / 1e9, 1), "TFLOP_per_s": round(flop / t / 1e12, 2),
                      "share_of_hbm_bound": round(nbytes / HBM_BW / t, 3), "share_of_fp32_bound": round(flop / FP32_PEAK / t, 3),
                      **info}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=436)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sea_raft.py measures on the GPU; no CUDA device found")
    info = card()
    for name in ("sea_raft_s", "sea_raft_l"):
        for dname in ("bf16", "fp16"):
            for batch in (4, 8):
                time_model(args, name, dname, batch, info)
    for dname in ("bf16", "fp16"):
        for batch in (4, 8):
            time_kernel(args, dname, batch, info)


if __name__ == "__main__":
    main()
