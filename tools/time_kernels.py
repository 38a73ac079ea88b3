"""Time this library's kernels alone, one named case at a time, on seeded inputs.

    python tools/time_kernels.py CASE [CASE ...] [--reps N] [--warmup 3] [--out RESULTS.jsonl]

A case sweeps its variants (shapes, storage types, implementations).  Each variant builds its inputs and returns the call to
time with the FLOP and the bytes it needs, counted from the shapes.  The call is timed with CUDA events over ``--reps``
launches (by default the case's own count), and one JSON line per variant gives the time, the achieved rates and the share of
the data-sheet peak that bounds it, beside the card's name, power limit and maximum SM clock.  A case can add one line that
sums its variants (skflow's six depthwise layers make one refinement iteration).  ``time_models.py`` runs the cases its
presets name after the models.
"""
from __future__ import annotations

import argparse
from typing import Callable, NamedTuple

import torch

import timing

DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16, "fp32": torch.float32}
GRID = (55, 128)  # the 1/8 grid of a 1024x436 pair


def _gen(seed: int = 0) -> torch.Generator:
    return torch.Generator(device="cuda").manual_seed(seed)


def attention_softmax_relpos(heads, mode, pairs=4, dtype="bf16"):
    """GMA's positional softmax at the 1024x436 grid.  Bytes: content logits read (position_and_content only), attention
    written, and the H + W fp32 table entries each row reads."""
    from ptlflow_b200 import ops

    (H, W), P, g = GRID, 160, _gen()
    N, npos, rows = H * W, 2 * P - 1, heads * pairs * H * W
    tables = torch.randn(rows, 640, device="cuda", generator=g)
    th, tw = tables[:, :npos], tables[:, npos:2 * npos]
    out = torch.empty(rows, N, dtype=DTYPES[dtype], device="cuda")
    logits = torch.randn(rows, N, device="cuda", generator=g).to(out.dtype) if mode == "position_and_content" else None
    nbytes = rows * N * out.element_size() * (2 if logits is not None else 1) + rows * (H + W) * 4
    return lambda: ops.attention_softmax_relpos(logits, th, tw, H, W, P, out=out), 0, nbytes


def depthwise_conv_gelu(layer, channels, k, pairs=8, dtype="bf16"):
    """SKFlow's depthwise convolution for one layer of the update block (``layer`` names it in the record).  FLOP = 2 k^2 C
    per pixel."""
    from ptlflow_b200 import ops

    (H, W), g = GRID, _gen()
    x = torch.randn(pairs, H, W, channels, device="cuda", generator=g).to(DTYPES[dtype])
    w, b = torch.randn(k * k, channels, device="cuda", generator=g) / k, torch.randn(channels, device="cuda", generator=g)
    out = torch.empty_like(x)
    return lambda: ops.depthwise_conv_gelu(x, w, b, k, out=out), 2.0 * k * k * channels * pairs * H * W, 0


def depthwise_conv_layernorm(dtype, pairs, channels=384, k=7):
    """SEA-RAFT's fused depthwise convolution + LayerNorm at the 1024x436 grid.  Bytes: one read of the input and one write of
    the output; FLOP = 2 k^2 C per pixel."""
    from ptlflow_b200 import ops

    (H, W), g = GRID, _gen(5)
    x = torch.randn(pairs, H, W, channels, device="cuda", generator=g).to(DTYPES[dtype])
    w = torch.randn(k * k, channels, device="cuda", generator=g) / k
    b = torch.randn(channels, device="cuda", generator=g) * 0.1
    out = torch.empty_like(x)
    P = pairs * H * W
    return lambda: ops.depthwise_conv_layernorm(x, w, b, k, out=out), 2.0 * k * k * channels * P, 2 * P * channels * x.element_size()


def attn1d(grid, axis, mode, impl, channels=256):
    """Flow1D's 1D attention or correlation along rows (axis 0) or columns (axis 1), one bf16 pair, on the wgmma or SIMT
    implementation.  FLOP per query and key: 4 C for an attention (q.k and p v), 2 C for a correlation."""
    from ptlflow_b200 import _lib, ops

    (h8, w8), g = grid, _gen()
    q, k, v = (torch.randn(1, h8, w8, channels, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3))
    m = _lib.ATTN1D_ATTN if mode == "attention" else _lib.ATTN1D_CORR
    v = v if m == _lib.ATTN1D_ATTN else None
    i = 2 if impl == "wgmma" else 1
    L = w8 if axis == 0 else h8
    flop = (4 if mode == "attention" else 2) * h8 * w8 * L * channels
    return lambda: ops.attn1d(q, k, v, axis, m, impl=i), flop, 0


def corr1d_lookup(grid, radius=32, stride=136, channels=256):
    """Flow1D's lookup in the row and column volumes, one bf16 pair.  Bytes: the lookup buffer written, the 2 (2r + 2) window
    values read per query and its coordinates."""
    from ptlflow_b200 import _lib, ops

    (h8, w8), g = grid, _gen()
    q, k = (torch.randn(1, h8, w8, channels, device="cuda", generator=g).to(torch.bfloat16) for _ in range(2))
    cx, cy = ops.attn1d(q, k, None, 0, _lib.ATTN1D_CORR), ops.attn1d(q, k, None, 1, _lib.ATTN1D_CORR)
    coords = (torch.rand(1, h8, w8, 2, device="cuda", generator=g) * torch.tensor([w8, h8], device="cuda")).contiguous()
    nbytes = h8 * w8 * (stride * 2 + 2 * (2 * radius + 2) * 2 + 8)
    return lambda: ops.corr1d_lookup(cx, cy, coords, radius, out_stride=stride), 0, nbytes


def knn_topk(grid, dtype, k=32, channels=256):
    """SCV's fused k-nearest-neighbour search, one pair; wgmma in bf16, SIMT in fp32.  FLOP = 2 N^2 C."""
    from ptlflow_b200 import ops

    (h, w), g = grid, _gen()
    f1, f2 = (torch.randn(1, h, w, channels, device="cuda", generator=g).to(DTYPES[dtype]) for _ in range(2))
    n = h * w
    return lambda: ops.knn_topk(f1, f2, k, channels ** -0.5), 2.0 * n * n * channels, 0


def sparse_lookup(grid=(112, 256), k=32, planes=408):
    """SCV's sparse-pyramid lookup at the 1/4 grid, bf16 output.  Bytes: the k-NN table and coordinates read, the planes
    written."""
    from ptlflow_b200 import ops

    (h, w), g = grid, _gen()
    n = h * w
    table = torch.randn(n, k, 3, device="cuda", generator=g) * 3
    coords = torch.zeros(1, h, w, 2, device="cuda")
    return lambda: ops.sparse_lookup(table, coords, torch.bfloat16, planes), 0, n * (k * 3 * 4 + 2 * 4 + planes * 2)


def shift_volume_tiled(dtype, pairs, levels=4):
    """LLA-Flow's shifted correlation volume (the GEMM with K = 26 x 256 and its pooled levels) at the 1024x436 grid.
    FLOP = 2 N^2 K per pair."""
    from ptlflow_b200 import ops

    (h8, w8), g = GRID, _gen()
    A = torch.randn(pairs, h8, w8, ops.LLA_K, device="cuda", generator=g).to(DTYPES[dtype])
    Bp = torch.randn(pairs, h8 + 4, w8 + 4, 512, device="cuda", generator=g).to(DTYPES[dtype])
    n = h8 * w8
    return lambda: ops.shift_volume_tiled(A, Bp, levels), 2.0 * n * n * ops.LLA_K * pairs, 0


def craft_volume_tiled(dtype, pairs, modes=4, levels=4):
    """CRAFT's fused inter-frame volume (clamp flag, statistics and the normalised tiled pyramid: three passes over the K = 256
    GEMM) at the 1024x436 grid.  FLOP = 3 x 2 N^2 256 per pair."""
    from ptlflow_b200 import ops

    (h8, w8), g = GRID, _gen()
    q1, k2 = (torch.randn(pairs, h8, w8, 256, device="cuda", generator=g).to(DTYPES[dtype]) for _ in range(2))
    bias = torch.randn(225, device="cuda", generator=g)
    n = h8 * w8
    return lambda: ops.craft_volume_tiled(q1, k2, modes, 0.5, bias, 7, levels), 3 * 2.0 * n * n * 256 * pairs, 0


def craft_window_softmax(modes, pairs, dtype="bf16"):
    """CRAFT's windowed-bias attention softmax over modes x pairs rows of N at the 1024x436 grid, in place.  Bytes: the logits read
    and the probabilities written."""
    from ptlflow_b200 import ops

    (h8, w8), g = GRID, _gen()
    n = h8 * w8
    x = torch.randn(modes * pairs * n, n, device="cuda", generator=g).to(DTYPES[dtype])
    bias = torch.randn(225, device="cuda", generator=g)
    flag = ops.craft_clamp_flag(x)
    return lambda: ops.craft_window_softmax(x, h8, w8, bias, 7, flag), 0, 2 * x.numel() * x.element_size()


def craft_mode_aggregate(F, modes, pairs, dtype="bf16"):
    """CRAFT's mode soft-aggregate + skip + LayerNorm at the 1024x436 grid (F = 256: the f2 transformer, 128: the loop's
    aggregator).  Bytes: the modes' features and the skip read, the result written."""
    from ptlflow_b200 import ops

    (h8, w8), g = GRID, _gen()
    feat = torch.randn(pairs, h8, w8, modes * F, device="cuda", generator=g).to(DTYPES[dtype])
    skip = torch.randn(pairs, h8, w8, F, device="cuda", generator=g).to(DTYPES[dtype])
    w = torch.randn(F, device="cuda", generator=g)
    out = torch.empty_like(skip)
    return lambda: ops.craft_mode_aggregate(feat, modes, w, 1.0, skip, out), 0, (feat.numel() + 2 * skip.numel()) * feat.element_size()


def softsplat_average(pairs, dtype="bf16", channels=128):
    """SplatFlow's average splat of the 128 motion channels (stride 256, as in the loop's motion buffer) into the mf_t columns of a
    256-channel buffer at the 1024x436 grid, by a random flow of a few px.  Bytes: source and flow read, the fp64 accumulator
    (channels + 1) cleared, added into and read once, the result written."""
    from ptlflow_b200 import ops

    (H, W), g = GRID, _gen(7)
    src = torch.randn(pairs, H, W, 2 * channels, device="cuda", generator=g).to(DTYPES[dtype])
    flow = 4 * torch.randn(pairs, 2, H, W, device="cuda", generator=g)
    out = torch.empty_like(src)
    P, es = pairs * H * W, src.element_size()
    nbytes = 2 * P * channels * es + P * 2 * 4 + 3 * P * (channels + 1) * 8
    return lambda: ops.softsplat_average(src, flow, out=out, channels=channels, out_offset=channels), 0, nbytes


class Case(NamedTuple):
    build: Callable  # (**variant) -> (fn, flop, nbytes)
    variants: list
    reps: int
    peak_flops: float = timing.PEAK_FLOPS
    total: str = ""  # when set, the label of one more record that sums the variants' times, FLOP and bytes


CASES = {
    "attention_softmax_relpos": Case(attention_softmax_relpos, [dict(heads=h, mode=m) for h in (1, 4)
                                                                for m in ("position_only", "position_and_content")], 50),
    # the depthwise steps of skflow's default update block, with padded channels (its k = 1 steps ride the ffn1 epilogue)
    "depthwise_conv_gelu": Case(depthwise_conv_gelu, [dict(layer=name, channels=c, k=k) for name, c, k in (
        ("encoder.convc1", 352, 15), ("encoder.convc2", 256, 15), ("encoder.convf2", 128, 15), ("encoder.conv", 256, 15), ("gru", 512, 7),
        ("flow_head", 128, 15))], 50, timing.PEAK_FLOPS_FP32, total="all per iteration"),
    "depthwise_conv_layernorm": Case(depthwise_conv_layernorm, [dict(dtype=d, pairs=b) for d in ("bf16", "f16") for b in (4, 8)], 50,
                                     timing.PEAK_FLOPS_FP32),
    "attn1d": Case(attn1d, [dict(grid=grid, axis=axis, mode=mode, impl=impl) for grid in (GRID, (270, 480)) for axis in (0, 1)
                            for mode in ("attention", "correlation") for impl in ("wgmma", "simt")], 20),
    "corr1d_lookup": Case(corr1d_lookup, [dict(grid=grid) for grid in (GRID, (270, 480))], 50),
    # N = 7 168 and 28 672; the 1/8 and 1/4 grids of a 1024x436 pair give 7 040 and 28 160
    "knn_topk": Case(knn_topk, [dict(grid=grid, dtype=d) for grid in ((56, 128), (112, 256)) for d in ("bf16", "fp32")], 10),
    "sparse_lookup": Case(sparse_lookup, [{}], 100),
    "shift_volume_tiled": Case(shift_volume_tiled, [dict(dtype=d, pairs=b) for d in ("bf16", "f16") for b in (1, 4)], 10),
    "craft_volume_tiled": Case(craft_volume_tiled, [dict(dtype=d, pairs=b) for d in ("bf16", "f16") for b in (1, 4)], 10),
    "craft_window_softmax": Case(craft_window_softmax, [dict(modes=4, pairs=b) for b in (1, 4)], 10),
    "craft_mode_aggregate": Case(craft_mode_aggregate, [dict(F=f, modes=4, pairs=b) for f in (128, 256) for b in (1, 4)], 50),
    "softsplat_average": Case(softsplat_average, [dict(pairs=b, dtype=d) for d in ("bf16", "f16") for b in (1, 4)], 50),
}


def run(name: str, reps: int = 0, warmup: int = 3, out: str = "") -> None:
    """Time every variant of case ``name`` (``reps`` launches each, 0 = the case's own count) and emit one record per variant."""
    case = CASES[name]
    total = [0.0, 0.0, 0.0]
    for variant in case.variants:
        fn, flop, nbytes = case.build(**variant)
        ms = timing.events_ms(fn, reps or case.reps, warmup)
        timing.emit({"kernel": name, **variant, "ms": round(ms, 4), **timing.bound_share(ms, flop, nbytes, peak_flops=case.peak_flops)}, out)
        total = [total[0] + ms, total[1] + flop, total[2] + nbytes]
        del fn
        torch.cuda.empty_cache()
    if case.total:
        timing.emit({"kernel": name, "variants": case.total, "ms": round(total[0], 4),
                     **timing.bound_share(*total, peak_flops=case.peak_flops)}, out)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("cases", nargs="+", choices=sorted(CASES), metavar="CASE", help=f"one or more of: {', '.join(CASES)}")
    ap.add_argument("--reps", type=int, default=0, help="launches per timing (default: the case's own count)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    a = ap.parse_args()
    for name in a.cases:
        run(name, a.reps, a.warmup, a.out)


if __name__ == "__main__":
    main()
