#!/usr/bin/env python
"""Streaming inference over a directory of frames: decode -> batches in flight -> flow files, all overlapped.

The caller-side loop of the reference (``infer.py``: ``cv.imread`` -> forward -> write, one pair at a time) rebuilt on
``ptlflow_b200.pipeline.FrameFeeder`` / ``FramePipeline`` and ``ptlflow_b200.utils.flow_utils.AsyncFlowWriter``
(SURVEY.md section 8(f) rank 4).  Needs a CUDA GPU; consecutive frames of the sorted directory listing form the pairs.

    python tools/infer_stream.py --model raft --ckpt things --frames /data/clip --out /data/clip_flow --batch 8
"""
import argparse
import os
import sys
import time
from pathlib import Path

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import ptlflow_b200 as pb  # noqa: E402
from ptlflow_b200.pipeline import FrameFeeder, FramePipeline  # noqa: E402
from ptlflow_b200.utils.flow_utils import AsyncFlowWriter  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="raft")
    ap.add_argument("--ckpt", default=None, help="checkpoint name or path, as for ptlflow.get_model")
    ap.add_argument("--frames", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--inflight", type=int, default=2)
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16", "fp32"])
    ap.add_argument("--format", default="flo", choices=["flo", "png", "npy"])
    a = ap.parse_args()

    files = sorted(p for p in Path(a.frames).iterdir() if p.suffix.lower() in (".png", ".jpg", ".jpeg", ".bmp", ".ppm"))
    pairs = list(zip(files[:-1], files[1:]))
    if not pairs:
        raise SystemExit(f"no frame pairs under {a.frames}")
    dtype = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}[a.dtype]
    model = pb.get_model(a.model, ckpt_path=a.ckpt).eval().cuda().to(dtype)
    os.makedirs(a.out, exist_ok=True)

    t0 = time.perf_counter()
    with FramePipeline(model, depth=a.inflight) as pipe, AsyncFlowWriter(workers=4) as writer:
        pending = []
        for idx, images in FrameFeeder(pairs, batch=a.batch, dtype=dtype):
            pending.append((idx, pipe.submit({"images": images})))
            while len(pending) > a.inflight:  # keep the queue short: results are written as soon as they are ready
                done_idx, res = pending.pop(0)
                flows = res.get()["flows"]  # [b,1,2,H,W]
                for j, i in enumerate(done_idx):
                    writer.submit(Path(a.out) / f"{pairs[i][0].stem}.{a.format}", flows[j, 0])
        for done_idx, res in pending:
            flows = res.get()["flows"]
            for j, i in enumerate(done_idx):
                writer.submit(Path(a.out) / f"{pairs[i][0].stem}.{a.format}", flows[j, 0])
    dt = time.perf_counter() - t0
    print(f"{len(pairs)} pairs in {dt:.2f} s = {len(pairs) / dt:.1f} pairs/s (decode, forward and write overlapped)")


if __name__ == "__main__":
    main()
