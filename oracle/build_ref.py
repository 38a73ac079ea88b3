#!/usr/bin/env python
"""Build the reference's own native plugin for this path, ``alt_cuda_corr`` (TEST INFRASTRUCTURE, see oracle/__init__.py).

The two source files are compiled where they lie under /root/reference (ptlflow/utils/external/alt_cuda_corr/
correlation.cpp + correlation_kernel.cu: plain CUDA C + a pybind11 shim, nothing arch specific) with
``torch.utils.cpp_extension`` for sm_90; only the resulting ``oracle/_ref/alt_cuda_corr.so`` is kept (git-ignored, it
sits next to the library build products).  No reference source is copied.

Uses: (1) the parity tests check ``ptlflow_b200.alt_cuda_corr.forward`` against the real reference kernel
(tests/test_gpu_ref_plugin.py), (2) tools/time_config4.py times it beside this library's on-the-fly kernel
(SURVEY.md section 8(d): the reference alt_cuda_corr as the existing native kernel comparator).
Where the reference checkout is absent nothing builds; a prebuilt file is only loaded.

    python oracle/build_ref.py            # -> oracle/_ref/alt_cuda_corr.so (a no-op when /root/reference is absent)
"""
from __future__ import annotations

import glob
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
SRC = "/root/reference/ptlflow/utils/external/alt_cuda_corr"
TARGET = os.path.join(OUT, "alt_cuda_corr.so")


def build(verbose: bool = False) -> str | None:
    if not os.path.isdir(SRC):
        return TARGET if os.path.exists(TARGET) else None
    srcs = [os.path.join(SRC, "correlation.cpp"), os.path.join(SRC, "correlation_kernel.cu")]
    if os.path.exists(TARGET) and all(os.path.getmtime(TARGET) >= os.path.getmtime(s) for s in srcs):
        return TARGET
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils import cpp_extension

    build_dir = os.path.join(OUT, "build_alt_cuda_corr")
    os.makedirs(build_dir, exist_ok=True)
    cpp_extension.load(name="alt_cuda_corr", sources=srcs, extra_cuda_cflags=["-O3"], build_directory=build_dir, verbose=verbose,
                       is_python_module=False)
    built = glob.glob(os.path.join(build_dir, "alt_cuda_corr*.so"))
    if not built:
        raise RuntimeError("alt_cuda_corr did not build")
    shutil.copy2(built[0], TARGET)
    shutil.rmtree(build_dir, ignore_errors=True)
    return TARGET


def load():
    """Import the prebuilt reference plugin (None when it was never built)."""
    if not os.path.exists(TARGET):
        return None
    import importlib.util

    import torch  # noqa: F401  (the extension links against libtorch)

    spec = importlib.util.spec_from_file_location("alt_cuda_corr", TARGET)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(verbose="--verbose" in sys.argv))
