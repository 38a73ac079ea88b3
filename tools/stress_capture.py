#!/usr/bin/env python
"""Stress the multi-threaded CUDA-graph capture path (needs a CUDA GPU): fresh models, two pipeline slots that see their shape for
the first and second time while the other slot is mid-forward, many rounds.  Prints full tracebacks of any failure.

    python tools/stress_capture.py [--rounds 12]
    PFB_CAPTURE_EXCLUSIVE=0 python tools/stress_capture.py     # without the forward / capture gate
"""
import argparse
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import ptlflow_b200 as pb  # noqa: E402
from ptlflow_b200.pipeline import FramePipeline  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=12)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    fails = 0
    for r in range(a.rounds):
        torch.manual_seed(r)
        model = pb.get_model("raft").eval().to(dev).half()
        model.iters = 4
        h, w = 128 + 8 * (r % 3), 192 + 16 * (r % 2)
        imgs = [torch.rand(2, 2, 3, h, w, device=dev).half() for _ in range(4)]
        # churn torch's stream pool the way a long test session does
        _ = [torch.cuda.Stream(device=dev) for _ in range(5 + r)]
        try:
            with torch.no_grad():
                ref = [model({"images": x})["flows"].float().cpu() for x in imgs]
            with FramePipeline(model, depth=2) as pipe:
                res = [pipe.submit({"images": imgs[k % 4]}) for k in range(12)]
                outs = [x.get()["flows"].float().cpu() for x in res]
            err = max((o - ref[k % 4]).abs().max().item() for k, o in enumerate(outs))
            print(f"round {r}: ok, max diff to sequential {err:.4f}", flush=True)
        except BaseException:  # noqa: BLE001
            fails += 1
            print(f"round {r}: FAILED", flush=True)
            traceback.print_exc()
            sys.stdout.flush()
            # a failed capture can leave the context unusable for this process
            try:
                torch.cuda.synchronize()
            except BaseException:  # noqa: BLE001
                print("context unusable after the failure; stopping", flush=True)
                break
    print(f"{fails} failed of {a.rounds}")


if __name__ == "__main__":
    main()
