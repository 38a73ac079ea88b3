"""Measuring code shared by the timing tools: the card a number was taken on, one CUDA-event timer, the per-kernel-class split
of an eager call, achieved rates against the data sheet, and one JSON line per record."""
from __future__ import annotations

import ctypes as C
import functools
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# NVIDIA's H100 SXM data sheet, for a card allowed up to 700 W: dense f16 / bf16 tensor-core rate, fp32 (non-tensor) rate, HBM3
PEAK_FLOPS = 989e12
PEAK_FLOPS_FP32 = 67e12
PEAK_BYTES = 3.35e12


@functools.lru_cache(maxsize=None)
def card() -> dict:
    """The card's name, power limit and maximum SM clock: a power-limited card runs below the data sheet's rates."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError) as e:
        reason = f"unknown ({type(e).__name__})"
        return {"gpu": torch.cuda.get_device_name(), "power_limit": reason, "max_sm_clock": reason}


def events_ms(fn, reps: int, warmup: int) -> float:
    """ms per call of ``fn``: ``warmup`` calls, a device synchronise, then CUDA events around ``reps`` calls."""
    if not torch.cuda.is_available():
        raise RuntimeError("events_ms times on a CUDA device and none was found")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / reps


def class_split(fn) -> dict:
    """{class name: {"ms", "launches"}} of this library's kernels in one eager call of ``fn`` (after one unprofiled call), for
    every class with launches."""
    from ptlflow_b200 import _lib

    lib = _lib.load()
    n = _lib.KERNEL_CLASSES
    ms, launches = (C.c_double * n)(), (C.c_ulonglong * n)()
    fn()
    torch.cuda.synchronize()
    _lib.check(lib.pfb_profile_enable(1), "profile_enable")
    try:
        fn()
        _lib.check(lib.pfb_profile_collect(ms, launches, n), "profile_collect")
    finally:
        lib.pfb_profile_enable(0)
    return {name: {"ms": round(ms[i], 3), "launches": int(launches[i])} for i, name in enumerate(_lib.KERNEL_CLASS_NAMES) if launches[i]}


def bound_share(ms: float, flop: float = 0, nbytes: float = 0, peak_flops: float = PEAK_FLOPS, peak_bytes: float = PEAK_BYTES) -> dict:
    """Achieved rates over ``ms``, and the share of peak: the least time the card could take (the larger of ``flop`` at
    ``peak_flops`` and ``nbytes`` at ``peak_bytes``) over ``ms``.  ``bound`` names the peak that set that least time."""
    t = ms * 1e-3
    compute, memory = flop / peak_flops, nbytes / peak_bytes
    return {"tflop_per_s": round(flop / t / 1e12, 2), "gb_per_s": round(nbytes / t / 1e9, 1),
            "share_of_peak": round(max(compute, memory) / t, 4),
            "bound": f"{peak_flops / 1e12:g} TFLOP/s" if compute >= memory else f"{peak_bytes / 1e12:g} TB/s"}


def emit(record: dict, out: str = "") -> None:
    """Print ``record`` with the card's fields as one JSON line, and append that line to ``out`` when given."""
    line = json.dumps({**record, **card()})
    print(line, flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "a") as f:
            f.write(line + "\n")
