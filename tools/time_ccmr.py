"""Time ccmr and ccmr_p at 1024x436 (default hyperparameters, random-init weights).

    python tools/time_ccmr.py [--steps 10] [--warmup 3] [--pairs 1 2] [--out results/time_ccmr.json]

Per model, dtype (bf16, f16) and pairs per step: CUDA events over ``--steps`` forwards after ``--warmup`` (each forward one CUDA-graph
launch), reported as ms per forward and pairs/s, next to the card name and its power limit read in the same run.  Then one eager bf16
forward of each model with the library's per-kernel-class timers.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from time_ms_raft import CLASSES, card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib

    lib = _lib.load()
    res = {"card": card(), "runs": [], "classes": {}}
    H, W = 436, 1024
    for name in ("ccmr", "ccmr_p"):
        base = pb.get_model(name).eval().cuda()
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
                run = {"model": name, "dtype": str(dtype).split(".")[-1], "pairs": b, "ms_per_forward": ms, "pairs_per_s": 1000.0 * b / ms,
                       "graph_replays": model.graph_replays}
                res["runs"].append(run)
                print(json.dumps(run), flush=True)
        model = base.to(torch.bfloat16)
        model.use_cuda_graph = False
        x = torch.rand(1, 2, 3, H, W, device="cuda", dtype=torch.bfloat16)
        with torch.no_grad():
            model({"images": x})
            torch.cuda.synchronize()
            lib.pfb_profile_enable(1)
            model({"images": x})
            ms = (C.c_double * _lib.KERNEL_CLASSES)()
            n = (C.c_ulonglong * _lib.KERNEL_CLASSES)()
            lib.pfb_profile_collect(ms, n, _lib.KERNEL_CLASSES)
            lib.pfb_profile_enable(0)
        res["classes"][name] = {CLASSES[i]: [round(ms[i], 3), int(n[i])] for i in range(_lib.KERNEL_CLASSES) if n[i]}
        print(name, "eager bf16 forward, ms and launches per kernel class:", res["classes"][name], flush=True)
        del base, model
        torch.cuda.empty_cache()
    print("card:", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
