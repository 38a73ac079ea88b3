"""Time scv4 and scv8 (default hyperparameters, random-init weights) beside raft at the same settings in the same process.

    python tools/time_scv.py [--steps 10] [--warmup 3] [--out results/time_scv.json]

1. Pairs/s at 1024x436 of scv4, scv8 and raft, bf16 and f16, 1 and 4 pairs per step, 12 and 32 iterations: CUDA events over
   ``--steps`` forwards after ``--warmup`` (each forward one CUDA-graph launch).
2. Peak allocated memory of one bf16 scv4 forward at 1024x436.
3. pfb_knn_topk alone on 56 x 128 and 112 x 256 grids (N = 7 168 and 28 672, C = 256; a 1024x436 pair gives 7 040 and 28 160) in
   bf16 and fp32: ms, TFLOP/s
   from 2 N^2 C per sample and the share of 989 TFLOP/s (the H100 SXM's dense f16 / bf16 rate; the kernel runs fp32 FMAs, whose
   rate is 67).
4. pfb_sparse_lookup alone on the 112 x 256 grid, k = 32, bf16 output: bytes moved from shapes (table + coordinates read, 408 channels
   written) and GB/s.
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


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import ptlflow_b200 as pb
    from ptlflow_b200 import ops

    res = {"card": card(), "runs": [], "knn": [], "lookup": {}}
    models = {name: pb.get_model(name).eval().cuda() for name in ("scv4", "scv8", "raft")}
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

    m = models["scv4"].to(torch.bfloat16)
    m.use_cuda_graph = False
    x = torch.rand(1, 2, 3, H, W, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        m({"images": x})
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        m({"images": x})
        torch.cuda.synchronize()
    res["scv4_peak_gib"] = round(torch.cuda.max_memory_allocated() / 2**30, 3)
    print("scv4 bf16 forward at 1024x436: peak allocated", res["scv4_peak_gib"], "GiB", flush=True)

    C = 256
    for grid, (h, w) in (("scv8", (56, 128)), ("scv4", (112, 256))):
        for dtype in (torch.bfloat16, torch.float32):
            f1 = torch.randn(1, h, w, C, device="cuda", dtype=dtype)
            f2 = torch.randn(1, h, w, C, device="cuda", dtype=dtype)
            ops.knn_topk(f1, f2, 32, C ** -0.5)
            ms = _events(lambda: ops.knn_topk(f1, f2, 32, C ** -0.5), a.steps)
            n = h * w
            tflops = 2.0 * n * n * C / ms / 1e9
            r = {"grid": grid, "N": n, "dtype": str(dtype).split(".")[-1], "ms": round(ms, 3), "tflops": round(tflops, 2),
                 "share_of_989": round(tflops / 989.0, 4)}
            res["knn"].append(r)
            print("knn_topk", json.dumps(r), flush=True)

    h, w, k = 112, 256, 32
    n = h * w
    table = torch.randn(n, k, 3, device="cuda") * 3
    coords = torch.zeros(1, h, w, 2, device="cuda")
    ops.sparse_lookup(table, coords, torch.bfloat16, 408)
    ms = _events(lambda: ops.sparse_lookup(table, coords, torch.bfloat16, 408), a.steps * 10)
    nbytes = n * (k * 3 * 4 + 2 * 4 + 408 * 2)
    res["lookup"] = {"N": n, "k": k, "ms": round(ms, 4), "bytes": nbytes, "gb_per_s": round(nbytes / ms / 1e6, 1)}
    print("sparse_lookup", json.dumps(res["lookup"]), flush=True)
    print("card:", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
