"""Time GMA's attention variants at the BASELINE config-3 per-GPU shape (1024x436, 12 iterations, bf16, 4 pairs per step).

    python tools/time_gma_variants.py [--batch 4] [--dtype bf16] [--steps 20] [--warmup 5] [--reps 50]

1. The model: ``gma`` with default hparams, position_only, position_and_content and num_heads=4 (random-init weights, seed
   1234, torch.rand frames, one CUDA graph launch per forward).  Pairs/s from CUDA events around --steps forwards after
   --warmup forwards (the first ones capture the graph).
2. pfb_attention_softmax_relpos alone at the same grid (55x128), 1 and 4 heads, both positional modes.  Bytes are computed
   from shapes: content logits read (position_and_content only) + attention written + the H + W table entries each row
   reads.  Kernel time from CUDA events around --reps back-to-back launches.

Prints one JSON line per measurement, each with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from argparse import Namespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VARIANTS = [("default", {}), ("position_only", {"position_only": True}), ("position_and_content", {"position_and_content": True}),
            ("num_heads=4", {"num_heads": 4})]


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


def time_models(args, dtype, info) -> None:
    import ptlflow_b200 as pb

    for name, hp in VARIANTS:
        torch.manual_seed(1234)
        model = pb.get_model("gma", args=Namespace(model=Namespace(iters=args.iters, **hp))).eval().cuda().to(dtype)
        frames = [torch.rand(args.batch, 2, 3, args.height, args.width, device="cuda").to(dtype) for _ in range(3)]
        step = [0]

        def fwd():
            model({"images": frames[step[0] % 3]})
            step[0] += 1

        with torch.no_grad():
            for _ in range(args.warmup):
                fwd()
            torch.cuda.synchronize()
            ms = events_ms(fwd, args.steps)
        print(json.dumps({"model": "gma", "hparams": hp or "default", "variant": name, "dtype": args.dtype, "batch": args.batch,
                          "image": [args.height, args.width], "iters": args.iters, "ms_per_step": round(ms, 3),
                          "pairs_per_s": round(args.batch / (ms * 1e-3), 1), "steps": args.steps, **info}), flush=True)
        del model, frames
        torch.cuda.empty_cache()


def time_kernel(args, dtype, info) -> None:
    from ptlflow_b200 import ops

    B, H, W, P = args.batch, -(-args.height // 8), -(-args.width // 8), 160
    N, npos = H * W, 2 * P - 1
    for heads in (1, 4):
        rows = heads * B * N
        tables = torch.randn(rows, 640, device="cuda")
        th, tw = tables[:, :npos], tables[:, npos:2 * npos]
        for mode in ("position_only", "position_and_content"):
            out = torch.empty(rows, N, dtype=dtype, device="cuda")
            logits = torch.randn(rows, N, device="cuda").to(dtype) if mode == "position_and_content" else None
            for _ in range(3):
                ops.attention_softmax_relpos(logits, th, tw, H, W, P, out=out)
            ms = events_ms(lambda: ops.attention_softmax_relpos(logits, th, tw, H, W, P, out=out), args.reps)
            nbytes = rows * N * out.element_size() * (2 if logits is not None else 1) + rows * (H + W) * 4
            print(json.dumps({"kernel": "pfb_attention_softmax_relpos", "mode": mode, "heads": heads, "batch": B, "grid": [H, W],
                              "dtype": args.dtype, "ms": round(ms, 4), "bytes": nbytes, "GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                              "hbm_peak_fraction_vs_3.35TBps": round(nbytes / (ms * 1e-3) / 3.35e12, 3), **info}), flush=True)
            del out, logits
        del tables
        torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--height", type=int, default=436)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=12)
    ap.add_argument("--dtype", default="bf16", choices=["fp16", "bf16", "fp32"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    dtype = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}[args.dtype]
    info = card()
    time_models(args, dtype, info)
    time_kernel(args, dtype, info)


if __name__ == "__main__":
    main()
