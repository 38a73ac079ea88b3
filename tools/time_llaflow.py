"""Time llaflow and llaflow_raft (default hyperparameters, random-init weights with both gammas set) beside gma and raft in the same process.

    python tools/time_llaflow.py [--steps 10] [--warmup 3] [--out results/time_llaflow.json]

1. Pairs/s at 1024x436 of llaflow, llaflow_raft, gma and raft, bf16 and f16, 1 and 4 pairs per step, 12 and 32 iterations: CUDA
   events over ``--steps`` forwards after ``--warmup`` (each forward one CUDA-graph launch).
2. The shifted-volume kernel (pfb_shift_volume_tiled, 4 levels) alone at the 1/8 grid of 1024x436 (128 x 55), 1 and 4 pairs, bf16 and
   f16: CUDA events over ``--steps`` launches, and its achieved TFLOP/s from the GEMM's 2 N^2 6656 FLOP per pair (N = 7040), with its
   share of the H100 SXM's 989 TFLOP/s dense f16 / bf16 peak.
The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from time_flow1d import _events  # noqa: E402
from time_ms_raft import card  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense f16 / bf16


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import ptlflow_b200 as pb
    from ptlflow_b200 import ops

    res = {"card": card(), "runs": [], "volume_kernel": []}
    models = {name: pb.get_model(name).eval().cuda() for name in ("llaflow", "llaflow_raft", "gma", "raft")}
    with torch.no_grad():
        for name in ("llaflow", "llaflow_raft"):  # both gammas are 0 at initialisation: give the new terms their real cost shape
            models[name].gamma.fill_(0.5)
            models[name].lsa.gamma.fill_(0.5)
    H, W = 436, 1024
    for iters in (12, 32):
        for dtype in (torch.bfloat16, torch.float16):
            for b in (1, 4):
                x = torch.rand(b, 2, 3, H, W, device="cuda", dtype=dtype)
                for name, base in models.items():
                    model = base.to(dtype)
                    model.iters = iters
                    with torch.no_grad():
                        for _ in range(a.warmup):
                            model({"images": x})
                        ms = _events(lambda: model({"images": x}), a.steps)
                    run = {"model": name, "size": f"{W}x{H}", "iters": iters, "dtype": str(dtype).split(".")[-1], "pairs": b,
                           "ms_per_forward": round(ms, 3), "pairs_per_s": round(1000.0 * b / ms, 2), "graph_replays": model.graph_replays}
                    res["runs"].append(run)
                    print(json.dumps(run), flush=True)
                    model._graphs.clear()
                    torch.cuda.empty_cache()

    h8, w8 = H // 8 + (H % 8 > 0), W // 8
    n = h8 * w8
    for dtype in (torch.bfloat16, torch.float16):
        for b in (1, 4):
            g = torch.Generator(device="cuda").manual_seed(0)
            A = torch.randn(b, h8, w8, ops.LLA_K, device="cuda", generator=g).to(dtype)
            Bp = torch.randn(b, h8 + 4, w8 + 4, 512, device="cuda", generator=g).to(dtype)
            for _ in range(a.warmup):
                ops.shift_volume_tiled(A, Bp, 4)
            ms = _events(lambda: ops.shift_volume_tiled(A, Bp, 4), a.steps)
            tflops = 2.0 * n * n * ops.LLA_K * b / (ms * 1e-3) / 1e12
            run = {"kernel": "pfb_shift_volume_tiled", "grid": f"{w8}x{h8}", "dtype": str(dtype).split(".")[-1], "pairs": b,
                   "ms": round(ms, 3), "tflops": round(tflops, 1), "share_of_dense_peak": round(tflops / PEAK_TFLOPS, 3)}
            res["volume_kernel"].append(run)
            print(json.dumps(run), flush=True)
            del A, Bp
            torch.cuda.empty_cache()
    print("card:", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
