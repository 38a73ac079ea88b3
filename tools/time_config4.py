#!/usr/bin/env python
"""BASELINE config 4 (raft, 1920x1080, 32 iterations, no 4D volume materialised) -- the lookup operator alone, timed three ways
on the same tensors (SURVEY.md section 8(d)): this library's on-the-fly kernel, the reference's own ``alt_cuda_corr`` built for
sm_90 (oracle/_ref, fp32 only like the reference uses it: corr.py:90-96), and this library's materialised-pyramid path
(volume build once + tiled lookup per iteration).  Prints one JSON line."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from oracle import build_ref  # noqa: E402
from ptlflow_b200 import ops  # noqa: E402

dev = "cuda:0"
B, H, W, C, L, R = 1, 135, 240, 256, 4, 4
torch.manual_seed(0)
f1 = torch.randn(B, H, W, C, device=dev)
f2 = torch.randn(B, H, W, C, device=dev)
ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
coords = (torch.stack([xs, ys], -1)[None] + 4.0 * torch.randn(B, H, W, 2, device=dev)).contiguous()


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


out = {"shape": f"1080p: {H}x{W} grid, C={C}, {L} levels, r={R}, one pair; ms per lookup of all levels (one refinement iteration)"}
for name, dt in (("ours_onthefly_fp32", torch.float32), ("ours_onthefly_f16", torch.float16)):
    a, b = f1.to(dt), f2.to(dt)
    pyr = ops.feature_pyramid(b, L)
    out[name] = round(timeit(lambda: ops.corr_lookup_onthefly(a, pyr, coords, R, nchw=False)), 4)
a16, b16 = f1.half(), f2.half()
pyr16 = ops.feature_pyramid(b16, L)
out["ours_onthefly_tensor_core_f16"] = round(timeit(lambda: ops.corr_lookup_onthefly_tc(a16, pyr16, coords, R)), 4)
o_tc = ops.corr_lookup_onthefly_tc(a16, pyr16, coords, R)
o_simt = ops.corr_lookup_onthefly(a16, pyr16, coords, R, nchw=False, out_stride=o_tc.shape[-1])
out["tensor_core_vs_simt_max_abs"] = float((o_tc[..., :L * 81].float() - o_simt[..., :L * 81].float()).abs().max())
out["tensor_core_flagged_queries"] = int(o_tc._pfb_flags.sum())
for sig in (1.0, 8.0):  # the same with smoother / rougher coordinates (the region GEMM serves fewer queries when the flow is rough)
    cs = (torch.stack([xs, ys], -1)[None] + sig * torch.randn(B, H, W, 2, device=dev)).contiguous()
    o = ops.corr_lookup_onthefly_tc(a16, pyr16, cs, R)
    out[f"ours_onthefly_tensor_core_f16_sigma{sig:g}"] = {"ms": round(timeit(lambda: ops.corr_lookup_onthefly_tc(a16, pyr16, cs, R)), 4), "flagged": int(o._pfb_flags.sum())}
ref = build_ref.load()
if ref is not None:
    pyr32 = ops.feature_pyramid(f2, L)

    def ref_all():  # what AlternateCorrBlock.__call__ does per iteration (corr.py:78-101): one kernel call per level
        return [ref.forward(f1, pyr32[l], (coords / 2**l)[:, None].contiguous(), R)[0] for l in range(L)]

    out["reference_alt_cuda_corr_fp32"] = round(timeit(ref_all, 5), 4)
    ours = ops.corr_lookup_onthefly(f1, pyr32, coords, R, nchw=True) * (C ** 0.5)
    refv = torch.cat([o[:, 0] for o in ref_all()], dim=1)
    out["max_abs_diff_vs_reference_kernel"] = float((ours - refv).abs().max())
t_build = timeit(lambda: ops.corr_volume_build_tiled(a16, b16, L), 5)
pyr_t = ops.corr_volume_build_tiled(a16, b16, L)
out["ours_materialised_f16"] = {"volume_build_once_ms": round(t_build, 4), "lookup_ms": round(timeit(lambda: ops.corr_lookup_tiled(pyr_t, coords, R, (H, W))), 4),
                                "pyramid_gb": round(sum(p.numel() * 2 for p in pyr_t) / 1e9, 3)}
print(json.dumps(out))
