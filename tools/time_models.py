"""Time the models' graphed forwards, and the kernels they added, from named presets.

    python tools/time_models.py PRESET [--steps N] [--warmup N] [--reps N] [--out RESULTS.jsonl]

Each model is built once per (model, hparams, dtype) with seed-1234 random-init weights, in eval mode on the GPU, then timed at
each of its runs: CUDA events over ``--steps`` forwards after ``--warmup`` (the first ones capture the CUDA graph, so the timed
forwards are one graph launch each), rotating three seeded frames.  Every run emits one JSON line with the same fields:
``model, hparams, dtype, pairs, size, iters, ms_per_forward, pairs_per_s, graph_replays`` (replays in this run), beside the
card's name, power limit and maximum SM clock.  Where the preset asks, one eager forward of a run adds the per-kernel-class split
(``split``) or a value derived from it.  Then the preset's kernel cases run (``time_kernels.py``).

Presets (1024x436 unless noted):
  gma_variants  gma with default, position_only, position_and_content and num_heads=4 hparams, bf16, 4 pairs, 12 iterations
  skflow        skflow, bf16 and f16, 4 and 8 pairs, 12 iterations, split
  sea_raft      sea_raft_s and sea_raft_l, bf16 and f16, 4 and 8 pairs, split with encoders / volume / loop_conv / dw_layernorm /
                other (the eager forward's event time minus those groups)
  ms_raft       ms_raft_p, bf16 and f16, 1, 2 and 4 pairs; split of bf16 at 1 pair with the loop's GFLOP and conv TFLOP/s
  ccmr          ccmr and ccmr_p, bf16 and f16, 1 and 2 pairs; split of bf16 at 1 pair
  flow1d        flow1d, 12 and 32 iterations, bf16 and f16, 1 and 4 pairs, and at 3840x2160 bf16 1 pair; split of bf16 at
                1 pair and 32 iterations
  csflow        csflow and raft, 12 and 32 iterations, bf16 and f16, 1 and 4 pairs; split of bf16 at 1 pair and 32 iterations;
                the strip channel's ms per iteration over raft
  scv           scv4, scv8 and raft, 12 and 32 iterations, bf16 and f16, 1 and 4 pairs; scv4's peak allocated memory
  llaflow       llaflow and llaflow_raft (both gammas at 0.5), gma and raft, 12 and 32 iterations, bf16 and f16, 1 and 4 pairs
"""
from __future__ import annotations

import argparse
import itertools
from argparse import Namespace
from typing import Callable, NamedTuple, Optional

import torch

import time_kernels
import timing

DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16, "fp32": torch.float32}


class Run(NamedTuple):
    model: str
    hparams: dict
    dtype: str
    pairs: int
    iters: Optional[int]  # None: the model's default
    size: str  # WxH


class Runs(NamedTuple):
    """Every combination of these values is one run."""
    models: tuple
    dtypes: tuple
    pairs: tuple
    iters: tuple = (None,)
    hparams: tuple = ({},)
    sizes: tuple = ("1024x436",)


class Preset(NamedTuple):
    runs: tuple  # of Runs
    steps: int
    warmup: int
    # (fields a run must match, fn(record, eager forward) -> fields added to its record): one eager forward's split, or a value
    # derived from it
    eager: tuple = ()
    kernels: tuple = ()  # names of time_kernels.CASES
    setup: dict = {}  # model name -> fn(model) before its runs
    summary: Optional[Callable] = None  # fn(records of all runs) -> one more record


def split(record, forward) -> dict:
    return {"split": timing.class_split(forward)}


def ms_raft_loop(record, forward) -> dict:
    """The split, and the update iterations' FLOP per pair counted from the layer shapes (the mask head, which runs in the last
    iteration only, excluded) over the time of the loop convolutions."""
    s = timing.class_split(forward)
    macs = 162 * 256 + 256 * 192 * 9 + 2 * 128 * 49 + 128 * 64 * 9 + 256 * 126 * 9  # motion encoder
    macs += 2 * 3 * 384 * 128 * 5  # SepConvGRU: z, r, q at 1x5 and 5x1 over [h | inp | motion]
    macs += 128 * 256 * 9 + 256 * 2 * 9  # flow head
    # 1024x436 padded to 1024x448; the loop runs at 1/16, 1/8, 1/4 and 1/2
    flop = sum(2.0 * macs * (448 // sc) * (1024 // sc) * it for sc, it in zip((16, 8, 4, 2), record["iters"]))
    return {"split": s, "loop_gflop": round(flop / 1e9, 1), "loop_conv_tflop_per_s": round(flop / (s["conv"]["ms"] * 1e-3) / 1e12, 1)}


SEA_RAFT_GROUPS = {"encoders": ("enc_affine", "enc_stats", "enc_conv1"), "volume": ("volume", "pool"),
                   "loop_conv": ("conv", "flowconv", "gather"), "dw_layernorm": ("dw_layernorm",)}


def sea_raft_groups(record, forward) -> dict:
    """The split, and its groups; other = the eager forward's event time minus the groups (cuDNN's encoder convolutions,
    lookup, upsample, copies, launch gaps)."""
    eager_ms = timing.events_ms(forward, 1, 1)
    s = timing.class_split(forward)
    groups = {g: round(sum(s[k]["ms"] for k in ks if k in s), 3) for g, ks in SEA_RAFT_GROUPS.items()}
    groups["other"] = round(eager_ms - sum(groups.values()), 3)
    return {"split": s, "eager_forward_ms": round(eager_ms, 3), "split_groups_ms": groups}


def peak_memory(record, forward) -> dict:
    """Peak memory allocated in the process during one eager forward."""
    forward()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    forward()
    torch.cuda.synchronize()
    return {"peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2**30, 3)}


def strip_ms_per_iteration(records) -> dict:
    """csflow's strip channel per iteration: (csflow - raft) at 32 iterations minus the same at 12, over 20."""
    ms = {(r["model"], r["iters"], r["dtype"], r["pairs"]): r["ms_per_forward"] for r in records}
    return {"strip_ms_per_iteration": {
        f"{d} x{b}": round(((ms["csflow", 32, d, b] - ms["raft", 32, d, b]) - (ms["csflow", 12, d, b] - ms["raft", 12, d, b])) / 20, 4)
        for d in ("bf16", "f16") for b in (1, 4)}}


def gammas_at_half(model) -> None:
    """Both gammas are 0 at initialisation: give the shift-aggregated terms their real cost shape."""
    model.gamma.fill_(0.5)
    model.lsa.gamma.fill_(0.5)


HALF = ("bf16", "f16")
BF16_1 = {"dtype": "bf16", "pairs": 1}
PRESETS = {
    "gma_variants": Preset(
        (Runs(("gma",), ("bf16",), (4,), (12,),
              ({}, {"position_only": True}, {"position_and_content": True}, {"num_heads": 4})),),
        steps=20, warmup=5, kernels=("attention_softmax_relpos",)),
    "skflow": Preset((Runs(("skflow",), HALF, (4, 8), (12,)),), steps=20, warmup=5, eager=(({}, split),),
                     kernels=("depthwise_conv_gelu",)),
    "sea_raft": Preset((Runs(("sea_raft_s", "sea_raft_l"), HALF, (4, 8)),), steps=20, warmup=5, eager=(({}, sea_raft_groups),),
                       kernels=("depthwise_conv_layernorm",)),
    "ms_raft": Preset((Runs(("ms_raft_p",), HALF, (1, 2, 4)),), steps=20, warmup=5, eager=((BF16_1, ms_raft_loop),)),
    "ccmr": Preset((Runs(("ccmr", "ccmr_p"), HALF, (1, 2)),), steps=10, warmup=3, eager=((BF16_1, split),)),
    "flow1d": Preset(
        (Runs(("flow1d",), HALF, (1, 4), (12, 32)), Runs(("flow1d",), ("bf16",), (1,), (12, 32), sizes=("3840x2160",))),
        steps=10, warmup=3, eager=(({**BF16_1, "iters": 32, "size": "1024x436"}, split),), kernels=("attn1d", "corr1d_lookup")),
    "csflow": Preset((Runs(("csflow", "raft"), HALF, (1, 4), (12, 32)),), steps=10, warmup=3,
                     eager=(({**BF16_1, "iters": 32}, split),), summary=strip_ms_per_iteration),
    "scv": Preset((Runs(("scv4", "scv8", "raft"), HALF, (1, 4), (12, 32)),), steps=10, warmup=3,
                  eager=(({"model": "scv4", **BF16_1, "iters": 32}, peak_memory),), kernels=("knn_topk", "sparse_lookup")),
    "llaflow": Preset((Runs(("llaflow", "llaflow_raft", "gma", "raft"), HALF, (1, 4), (12, 32)),), steps=10, warmup=3,
                      kernels=("shift_volume_tiled",), setup={"llaflow": gammas_at_half, "llaflow_raft": gammas_at_half}),
}


def matches(run: Run, fields: dict) -> bool:
    return all(getattr(run, k) == v for k, v in fields.items())


def _model_key(run: Run) -> str:
    return repr((run.model, sorted(run.hparams.items()), run.dtype))  # (hparams is a dict, so not hashable itself)


def expand(preset: Preset) -> list:
    """The preset's runs, those of one (model, hparams, dtype) next to each other (they share one model)."""
    runs = [Run(m, hp, d, b, it, size) for g in preset.runs
            for m, hp, d, b, it, size in itertools.product(g.models, g.hparams, g.dtypes, g.pairs, g.iters, g.sizes)]
    first = {}
    for r in runs:
        first.setdefault(_model_key(r), len(first))
    return sorted(runs, key=lambda r: first[_model_key(r)])


def time_model(preset: Preset, runs: list, steps: int, warmup: int, out: str) -> list:
    """Build the model of ``runs`` (one model, hparams and dtype), time each run and emit its record."""
    import ptlflow_b200 as pb

    name, hparams, dname = runs[0].model, runs[0].hparams, runs[0].dtype
    torch.manual_seed(1234)
    model = pb.get_model(name, args=Namespace(model=Namespace(**hparams))).eval().cuda().to(DTYPES[dname])
    records = []
    with torch.no_grad():
        if name in preset.setup:
            preset.setup[name](model)
        for run in runs:
            if run.iters is not None:
                model.iters = run.iters
            W, H = map(int, run.size.split("x"))
            g = torch.Generator(device="cuda").manual_seed(0)
            frames = [torch.rand(run.pairs, 2, 3, H, W, device="cuda", generator=g).to(DTYPES[dname]) for _ in range(3)]
            step = itertools.count()

            def forward():
                model({"images": frames[next(step) % 3]})

            replays = model.graph_replays
            ms = timing.events_ms(forward, steps, warmup)
            record = {"model": name, "hparams": hparams, "dtype": dname, "pairs": run.pairs, "size": run.size, "iters": model.iters,
                      "ms_per_forward": round(ms, 3), "pairs_per_s": round(run.pairs / (ms * 1e-3), 2),
                      "graph_replays": model.graph_replays - replays}
            for fields, fn in preset.eager:
                if matches(run, fields):
                    graphed, model.use_cuda_graph = model.use_cuda_graph, False
                    try:
                        record.update(fn(record, forward))
                    finally:
                        model.use_cuda_graph = graphed
            timing.emit(record, out)
            records.append(record)
            del frames, forward
    del model
    torch.cuda.empty_cache()
    return records


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("preset", choices=sorted(PRESETS))
    ap.add_argument("--steps", type=int, help="timed forwards per run (default: the preset's)")
    ap.add_argument("--warmup", type=int, help="forwards before the timed ones, and launches before a kernel's (default: the preset's)")
    ap.add_argument("--reps", type=int, default=0, help="launches per kernel timing (default: each case's own count)")
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    a = ap.parse_args()
    preset = PRESETS[a.preset]
    steps = a.steps or preset.steps
    warmup = preset.warmup if a.warmup is None else a.warmup
    records = []
    for _, runs in itertools.groupby(expand(preset), key=_model_key):
        records += time_model(preset, list(runs), steps, warmup, a.out)
    if preset.summary is not None:
        timing.emit({"preset": a.preset, **preset.summary(records)}, a.out)
    for name in preset.kernels:
        time_kernels.run(name, a.reps, warmup, a.out)


if __name__ == "__main__":
    main()
