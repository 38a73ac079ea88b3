"""Time lcv_raft beside raft and lcv_raft_small beside raft_small, and the tiled lookup on a frozen pyramid.

    python tools/time_lcv.py [--steps 10] [--warmup 3] [--out RESULTS.jsonl]

At 1024x436, bf16 and f16, 1 and 4 pairs, 12 and 32 iterations, one CUDA graph per forward: each model is built once per dtype with
seed-1234 random-init weights (for LCV, W = I: the fold's cost does not depend on its values) and timed as tools/time_models.py
times its runs (CUDA events over ``--steps`` graphed forwards, three seeded inputs rotating); one JSON line per run gives ``model,
dtype, pairs, iters, ms_per_forward, pairs_per_s`` beside the card's name and power limit.  First the lookup kernel's time (time_lookup: launches
replayed from a CUDA graph) at the 55x128 grid of 1024x436 frames with RAFT's pyramid and with explicit level sizes (the same sizes:
at 55x128 every level pools), and on the 17x21 grid of 136x168 frames with LCV's frozen levels.  ``--lookup-only`` times only
pfb_corr_lookup_tiled at 55x128, which every build of the library has: run it from an older tree to compare builds.
"""
from __future__ import annotations

import argparse
import itertools
from argparse import Namespace

import torch

import timing

DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}
H, W = 436, 1024


def time_runs(name: str, dname: str, steps: int, warmup: int, out: str) -> None:
    import ptlflow_b200 as pb

    torch.manual_seed(1234)
    model = pb.get_model(name, args=Namespace(model=Namespace())).eval().cuda().to(DTYPES[dname])
    with torch.no_grad():
        for pairs, iters in itertools.product((1, 4), (12, 32)):
            model.iters = iters
            g = torch.Generator(device="cuda").manual_seed(0)
            inputs = [torch.rand(pairs, 2, 3, H, W, device="cuda", generator=g).to(DTYPES[dname]) for _ in range(3)]
            step = itertools.count()

            def forward():
                model({"images": inputs[next(step) % 3]})

            ms = timing.events_ms(forward, steps, warmup)
            timing.emit({"model": name, "dtype": dname, "pairs": pairs, "size": f"{W}x{H}", "iters": iters,
                         "ms_per_forward": round(ms, 3), "pairs_per_s": round(pairs / (ms * 1e-3), 2)}, out)
            del inputs, forward
    del model
    torch.cuda.empty_cache()


def time_lookup(grid, explicit: bool, out: str, graph_calls: int = 100, replays: int = 20) -> None:
    """Kernel time of the tiled lookup (radius 4, 4 levels, bf16, one pair) on the loop's pyramid: ``graph_calls`` raw C calls into one
    preallocated output, captured as one CUDA graph and replayed ``replays`` times between CUDA events, so neither the Python wrapper
    nor the host's launch rate is in the time.  ``explicit``: pfb_corr_lookup_tiled_ex with LCV's level sizes (2r+1 = 9), else
    pfb_corr_lookup_tiled with RAFT's.  Needs only what the library had before pfb_corr_lookup_tiled_ex when ``explicit`` is False."""
    import ctypes as C

    from ptlflow_b200 import _lib, ops

    lib = _lib.load()
    h, w = grid
    sizes = [(h >> l, w >> l) for l in range(4)]
    if explicit:
        sizes, distinct = ops.corr_level_sizes(h, w, 4, 9)
    else:
        distinct = 4
    f = torch.randn(1, h, w, 256, device="cuda").to(torch.bfloat16)
    pyr = ops.corr_volume_build_tiled(f, f, distinct)
    pyr = pyr + [pyr[-1]] * (4 - distinct)
    coords = (torch.stack(torch.meshgrid(torch.arange(w), torch.arange(h), indexing="xy"), -1).float().cuda()[None]
              + torch.randn(1, h, w, 2, device="cuda")).contiguous()
    res = torch.empty((1, h, w, 328), dtype=torch.bfloat16, device="cuda")
    ptrs = _lib.ptr_array(pyr)
    lh, lw = (C.c_int * 4)(*[s[0] for s in sizes]), (C.c_int * 4)(*[s[1] for s in sizes])
    dt = _lib.dtype_code(torch.bfloat16)

    def call():
        s = _lib.stream_ptr()
        if explicit:
            rc = lib.pfb_corr_lookup_tiled_ex(ptrs, lh, lw, coords.data_ptr(), res.data_ptr(), 1, h, w, h, w, 4, 4, dt, 328, s)
        else:
            rc = lib.pfb_corr_lookup_tiled(ptrs, coords.data_ptr(), res.data_ptr(), 1, h, w, h, w, 4, 4, dt, 328, s)
        _lib.check(rc, "corr_lookup_tiled")

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            call()
        side.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=side):
            for _ in range(graph_calls):
                call()
    torch.cuda.current_stream().wait_stream(side)
    ms = timing.events_ms(graph.replay, replays, 3)
    timing.emit({"kernel": "corr_lookup_tiled_ex" if explicit else "corr_lookup_tiled", "grid": f"{h}x{w}",
                 "levels": [list(s) for s in sizes], "us_per_kernel": round(ms * 1e3 / graph_calls, 2),
                 "timed": f"{graph_calls} launches per CUDA graph, {replays} replays"}, out)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    ap.add_argument("--lookup-only", action="store_true", help="only the lookup kernel at 55x128 with RAFT's sizes (runs on older builds)")
    a = ap.parse_args()
    if a.lookup_only:
        time_lookup((55, 128), False, a.out)
        return
    time_lookup((55, 128), False, a.out)
    time_lookup((55, 128), True, a.out)
    time_lookup((17, 21), True, a.out)
    for dname in DTYPES:
        for name in ("raft", "lcv_raft", "raft_small", "lcv_raft_small"):
            time_runs(name, dname, a.steps, a.warmup, a.out)


if __name__ == "__main__":
    main()
