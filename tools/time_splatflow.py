"""Time splatflow with two and three frames beside gma, and its splat kernel.

    python tools/time_splatflow.py [--steps 10] [--warmup 3] [--out RESULTS.jsonl]

At 1024x436, bf16 and f16, 1 and 4 pairs, 12 and 32 iterations: ``splatflow`` fed T = 2 frames (pair (0, 1)) and T = 3 frames
(pairs (0, 1) and (1, 2), one CUDA graph), and ``gma`` (one head) on the same pair count.  Each model is built once per dtype with
seed-1234 random-init weights and timed as tools/time_models.py times its runs (CUDA events over ``--steps`` graphed forwards,
three seeded inputs rotating); one JSON line per run gives ``model, frames, dtype, pairs, iters, ms_per_forward, pairs_per_s``
(output pairs: one per sample) and ``peak_gib``, the peak allocated memory of one eager forward, beside the card's name and power
limit.  Then the ``softsplat_average`` kernel case of tools/time_kernels.py.
"""
from __future__ import annotations

import argparse
import itertools
from argparse import Namespace

import torch

import time_kernels
import timing

DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}
H, W = 436, 1024


def time_runs(name: str, frames: int, dname: str, steps: int, warmup: int, out: str) -> None:
    import ptlflow_b200 as pb

    torch.manual_seed(1234)
    model = pb.get_model(name, args=Namespace(model=Namespace())).eval().cuda().to(DTYPES[dname])
    with torch.no_grad():
        for pairs, iters in itertools.product((1, 4), (12, 32)):
            model.iters = iters
            g = torch.Generator(device="cuda").manual_seed(0)
            inputs = [torch.rand(pairs, frames, 3, H, W, device="cuda", generator=g).to(DTYPES[dname]) for _ in range(3)]
            step = itertools.count()

            def forward():
                model({"images": inputs[next(step) % 3]})

            ms = timing.events_ms(forward, steps, warmup)
            graphed, model.use_cuda_graph = model.use_cuda_graph, False
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            forward()
            torch.cuda.synchronize()
            model.use_cuda_graph = graphed
            timing.emit({"model": name, "frames": frames, "dtype": dname, "pairs": pairs, "size": f"{W}x{H}", "iters": iters,
                         "ms_per_forward": round(ms, 3), "pairs_per_s": round(pairs / (ms * 1e-3), 2),
                         "peak_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)}, out)
            del inputs, forward
    del model
    torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    a = ap.parse_args()
    for dname in DTYPES:
        for name, frames in (("splatflow", 2), ("splatflow", 3), ("gma", 2)):
            time_runs(name, frames, dname, a.steps, a.warmup, a.out)
    time_kernels.run("softsplat_average", 0, a.warmup, a.out)


if __name__ == "__main__":
    main()
