"""Time csflow (default hyperparameters, random-init weights) beside raft at the same settings in the same process.

    python tools/time_csflow.py [--steps 10] [--warmup 3] [--out results/time_csflow.json]

1. Pairs/s at 1024x436 of csflow and raft, bf16 and f16, 1 and 4 pairs per step, 12 and 32 iterations: CUDA events over ``--steps``
   forwards after ``--warmup`` (each forward one CUDA-graph launch).  The per-iteration cost of the strip channel is
   (csflow ms - raft ms) at 32 iterations minus the same at 12, over 20.
2. One eager bf16 forward at 1024x436, 32 iterations, of each model with the library's per-kernel-class timers (the strip lookup
   counts as lookup, pfb_strip_means and pfb_strip_prepare as misc).
The card's name and power limit are read in the same run.
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

from time_flow1d import _events  # noqa: E402
from time_ms_raft import CLASSES, card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib

    lib = _lib.load()
    res = {"card": card(), "runs": [], "classes": {}}
    models = {name: pb.get_model(name).eval().cuda() for name in ("csflow", "raft")}
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

    def ms_of(name, iters, dtype, b):
        return next(r["ms_per_forward"] for r in res["runs"] if (r["model"], r["iters"], r["dtype"], r["pairs"]) == (name, iters, dtype, b))

    res["strip_ms_per_iteration"] = {
        f"{dt} x{b}": round(((ms_of("csflow", 32, dt, b) - ms_of("raft", 32, dt, b)) - (ms_of("csflow", 12, dt, b) - ms_of("raft", 12, dt, b))) / 20, 4)
        for dt in ("bfloat16", "float16") for b in (1, 4)}
    print("strip channel, ms per iteration over raft:", res["strip_ms_per_iteration"], flush=True)

    x = torch.rand(1, 2, 3, H, W, device="cuda", dtype=torch.bfloat16)
    for name, base in models.items():
        model = base.to(torch.bfloat16)
        model.iters, model.use_cuda_graph = 32, False
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
        print(f"{name}: eager bf16 forward at 1024x436, 32 iterations, ms and launches per kernel class:", res["classes"][name], flush=True)
    print("card:", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
