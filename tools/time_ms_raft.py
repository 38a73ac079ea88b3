"""Time ms_raft_p at 1024x436 (default hyperparameters, random-init weights) and split one eager forward by kernel class.

    python tools/time_ms_raft.py [--steps 20] [--warmup 5] [--pairs 1 2 4] [--out results/time_ms_raft.json]

Per dtype (bf16, f16) and pairs per step: CUDA events over ``--steps`` forwards after ``--warmup`` (each forward one CUDA-graph
launch), reported as ms per forward and pairs/s, next to the card name and its power limit read in the same run.  Then one eager bf16
forward with the library's per-kernel-class timers, and the loop convolutions' TFLOP/s with FLOPs counted from the layer shapes.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CLASSES = ["volume", "pool", "lookup", "onthefly", "conv", "upsample", "misc", "enc_affine", "enc_stats", "enc_conv1", "flowconv",
           "gather", "depthwise", "dw_layernorm", "attn1d"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (power limit unavailable: {e})"


def loop_flops_per_pixel(planes: int = 162) -> float:
    """Multiply-adds x 2 of one update iteration per grid pixel, from the layer shapes (mask head excluded: last iteration only)."""
    macs = planes * 256 + 256 * 192 * 9 + 2 * 128 * 49 + 128 * 64 * 9 + 256 * 126 * 9  # motion encoder
    macs += 2 * 3 * 384 * 128 * 5  # SepConvGRU: z, r, q at 1x5 and 5x1 over [h | inp | motion]
    macs += 128 * 256 * 9 + 256 * 2 * 9  # flow head
    return 2.0 * macs


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--pairs", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib

    lib = _lib.load()
    res = {"card": card(), "runs": []}
    H, W = 436, 1024
    base = pb.get_model("ms_raft_p").eval().cuda()
    for dtype in (torch.bfloat16, torch.float16):
        model = base.to(dtype)
        for b in a.pairs:
            x = torch.rand(b, 2, 3, H, W, device="cuda", dtype=dtype)
            with torch.no_grad():
                for _ in range(a.warmup):
                    model({"images": x})
                torch.cuda.synchronize()
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                for _ in range(a.steps):
                    model({"images": x})
                t1.record()
                torch.cuda.synchronize()
            ms = t0.elapsed_time(t1) / a.steps
            res["runs"].append({"dtype": str(dtype)[6:], "pairs": b, "ms_per_forward": ms, "pairs_per_s": 1000.0 * b / ms,
                                "graph_replays": model.graph_replays})
            print(json.dumps(res["runs"][-1]), flush=True)
    # per-class split of one eager forward (bf16, 1 pair)
    model = base.to(torch.bfloat16)
    model.use_cuda_graph = False
    x = torch.rand(1, 2, 3, H, W, device="cuda", dtype=torch.bfloat16)
    n = _lib.KERNEL_CLASSES
    ms, cnt = (C.c_double * n)(), (C.c_ulonglong * n)()
    with torch.no_grad():
        model({"images": x})
        torch.cuda.synchronize()
        lib.pfb_profile_enable(1)
        model({"images": x})
        lib.pfb_profile_collect(ms, cnt, n)
        lib.pfb_profile_enable(0)
    split = {CLASSES[i]: round(ms[i], 3) for i in range(n) if cnt[i]}
    hp, wp = 448, 1024
    flops = sum(loop_flops_per_pixel() * (hp // s) * (wp // s) * it for s, it in zip((16, 8, 4, 2), model.iters))
    res["eager_split_ms"] = split
    res["loop_gflop"] = flops / 1e9
    res["loop_conv_tflops"] = flops / (split.get("conv", float("nan")) * 1e-3) / 1e12 if split.get("conv") else None
    print(json.dumps({k: v for k, v in res.items() if k != "runs"}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
