"""Build libptlflow_b200.so in-tree with nvcc for sm_90a (H100) (no torch involved).

    python -m ptlflow_b200.csrc.build [--force] [--verbose]

The .so and its build stamp land in ptlflow_b200/lib/ (both git-ignored).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
ROOT = os.path.dirname(PKG)
LIB_DIR = os.path.join(PKG, "lib")
OBJ_DIR = os.path.join(HERE, "build")
LIB_PATH = os.path.join(LIB_DIR, "libptlflow_b200.so")

SOURCES = ["misc.cu", "prof.cu", "corr.cu", "conv_simt.cu", "refine.cu", "conv_umma.cu", "corr_umma.cu", "corr_tiled.cu", "corr_onthefly_umma.cu", "conv_special.cu", "tmap.cu", "encoder.cu", "first_conv.cu", "depthwise.cu", "skflow.cu", "searaft.cu", "msraft.cu", "ccmr.cu", "enc_conv_umma.cu", "attn1d.cu", "csflow.cu", "scv.cu", "knn_umma.cu", "llaflow.cu", "craft.cu", "splatflow.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest() -> str:
    h = hashlib.sha256()
    for name in sorted(os.listdir(HERE)) + [os.path.join(ROOT, "include", "ptlflow_b200.h")]:
        path = name if os.path.isabs(name) else os.path.join(HERE, name)
        if path.endswith((".cu", ".cuh", ".h", "build.py")):
            with open(path, "rb") as f:
                h.update(name.encode() + b"\0" + f.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    stamp = os.path.join(LIB_DIR, "build.stamp")
    digest = _digest()
    if not force and os.path.exists(LIB_PATH) and os.path.exists(stamp) and open(stamp).read().strip() == digest:
        return LIB_PATH
    nvcc = _nvcc()

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-I", os.path.join(ROOT, "include"), "-c", os.path.join(HERE, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and r.stderr:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", LIB_PATH, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
