"""Time flow1d (default hyperparameters, random-init weights) and its two new kernels.

    python tools/time_flow1d.py [--steps 10] [--warmup 3] [--out results/time_flow1d.json]

1. Pairs/s at 1024x436 for 12 and 32 iterations, bf16 and f16, 1 and 4 pairs per step, and at 3840x2160 (1 pair, bf16, 12 and 32
   iterations): CUDA events over ``--steps`` forwards after ``--warmup`` (each forward one CUDA-graph launch).
2. One eager bf16 forward at 1024x436 with the library's per-kernel-class timers.
3. pfb_attn1d alone on the shapes of that forward (each attention and both correlations), and pfb_corr1d_lookup alone: CUDA events
   over repeated launches; FLOP = 2 L C per query and key for a correlation, 4 L C for an attention (q.k and p v); lookup bytes =
   the unique bytes from the shapes: the lookup buffer written, the 2 (2r+2) window values read per query (2 bytes each) and its
   coordinates (8 bytes).  The attention kernel is timed on both implementations (wgmma and SIMT).  Each is reported against 989 TFLOP/s (dense f16 / bf16 tensor core)
   and 3.35 TB/s (HBM3), the H100 SXM data sheet's figures at 700 W.
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

from time_ms_raft import CLASSES, card  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12


def _events(fn, reps: int) -> float:
    """ms per call of fn over reps calls after one warm-up."""
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import ptlflow_b200 as pb
    from ptlflow_b200 import _lib, ops

    lib = _lib.load()
    res = {"card": card(), "runs": [], "classes": {}, "kernels": []}
    base = pb.get_model("flow1d").eval().cuda()
    runs = [(436, 1024, it, dt, b) for it in (12, 32) for dt in (torch.bfloat16, torch.float16) for b in (1, 4)]
    runs += [(2160, 3840, it, torch.bfloat16, 1) for it in (12, 32)]
    for H, W, iters, dtype, b in runs:
        model = base.to(dtype)
        model.iters = iters
        x = torch.rand(b, 2, 3, H, W, device="cuda", dtype=dtype)
        with torch.no_grad():
            for _ in range(a.warmup):
                model({"images": x})
            ms = _events(lambda: model({"images": x}), a.steps)
        run = {"size": f"{W}x{H}", "iters": iters, "dtype": str(dtype).split(".")[-1], "pairs": b, "ms_per_forward": round(ms, 3),
               "pairs_per_s": round(1000.0 * b / ms, 2), "graph_replays": model.graph_replays}
        res["runs"].append(run)
        print(json.dumps(run), flush=True)
        model._graphs.clear()
        torch.cuda.empty_cache()

    model = base.to(torch.bfloat16)
    model.iters, model.use_cuda_graph = 32, False
    x = torch.rand(1, 2, 3, 436, 1024, device="cuda", dtype=torch.bfloat16)
    with torch.no_grad():
        model({"images": x})
        torch.cuda.synchronize()
        lib.pfb_profile_enable(1)
        model({"images": x})
        ms = (C.c_double * _lib.KERNEL_CLASSES)()
        n = (C.c_ulonglong * _lib.KERNEL_CLASSES)()
        lib.pfb_profile_collect(ms, n, _lib.KERNEL_CLASSES)
        lib.pfb_profile_enable(0)
    res["classes"] = {CLASSES[i]: [round(ms[i], 3), int(n[i])] for i in range(_lib.KERNEL_CLASSES) if n[i]}
    print("eager bf16 forward at 1024x436, 32 iterations, ms and launches per kernel class:", res["classes"], flush=True)

    # the kernels alone, on the 1/8 grid of 1024x436 (55 x 128) and of 3840x2160 (270 x 480), one pair, bf16
    g = torch.Generator(device="cuda").manual_seed(0)
    for h8, w8 in ((55, 128), (270, 480)):
        q, k, v = (torch.randn(1, h8, w8, 256, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3))
        P = h8 * w8
        for axis in (0, 1):
            L = w8 if axis == 0 else h8
            for mode, name, per in ((_lib.ATTN1D_ATTN, "attention", 4), (_lib.ATTN1D_CORR, "correlation", 2)):
                for impl, path in ((2, "wgmma"), (1, "simt")):
                    t = _events(lambda: ops.attn1d(q, k, v if mode == _lib.ATTN1D_ATTN else None, axis, mode, impl=impl), 20)
                    flops = per * P * L * 256
                    r = {"kernel": f"attn1d {name} axis {axis} {path}", "grid": f"{h8}x{w8}", "L": L, "ms": round(t, 4),
                         "tflops": round(flops / t / 1e9, 2), "share_of_989": round(flops / t / 1e-3 / PEAK_FLOPS, 4)}
                    res["kernels"].append(r)
                    print(json.dumps(r), flush=True)
        cx, cy = ops.attn1d(q, k, None, 0, _lib.ATTN1D_CORR), ops.attn1d(q, k, None, 1, _lib.ATTN1D_CORR)
        coords = (torch.rand(1, h8, w8, 2, device="cuda", generator=g) * torch.tensor([w8, h8], device="cuda")).contiguous()
        radius, stride = 32, 136
        t = _events(lambda: ops.corr1d_lookup(cx, cy, coords, radius, out_stride=stride), 50)
        nbytes = P * (stride * 2 + 2 * (2 * radius + 2) * 2 + 8)
        r = {"kernel": "corr1d_lookup r=32", "grid": f"{h8}x{w8}", "ms": round(t, 4), "gb_per_s": round(nbytes / t / 1e6, 1),
             "share_of_3.35TB": round(nbytes / t / 1e-3 / PEAK_BYTES, 4)}
        res["kernels"].append(r)
        print(json.dumps(r), flush=True)
    print("card:", res["card"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
