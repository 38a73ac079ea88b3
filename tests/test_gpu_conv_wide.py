"""Conformance of the convolution's 256-pixel work item (conv_wide_kernel in csrc/conv_umma.cu) against the float64
reference of conv_reference.py, with the per-element bounds and sentinel checks of test_gpu_conv_conformance.py.

The 256-pixel kernel takes the 3x3 layers with at least 128 input channels, an N tile of 96 or 128 and a ReLU epilogue
(with or without the two flow columns) on grids whose 128-pixel rows waste at most 30 % of the width.  The cases below
reach it by their shape alone: odd heights (an item whose second row lies below the image), widths that are and are not
multiples of 128, batches whose last CTA round is partial, an N tile of 96 with its 32-channel last block, several N tiles
and an output offset.  test_cases_take_the_wide_kernel checks from the launch trace that each of them ran on it."""
import json
import os
import subprocess
import sys

import pytest
import torch

import conv_reference as R
from test_gpu_conv_conformance import _report, case, run

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF = [torch.float16, torch.bfloat16]

CASES = [
    # RAFT's flow1 / mask1 form: 128 -> 256, two N tiles of 128; odd height, 3 x 4 x 1 = 12 items per N tile
    case("wide_nt128_x2_odd_h", 3, 7, 128, (3, 3), [(128,)], 256, R.RELU),
    # RAFT's convc2 form: 256 -> 192, two N tiles of 96 (a 64-channel TMA block + a 32-channel block each); width 200
    # (two 128-pixel rows, the second clipped at 72), out_offset 8 inside a wider pixel stride
    case("wide_nt96_x2_w200", 2, 5, 200, (3, 3), [(256,)], 192, R.RELU, out_offset=8),
    # RAFT's conv form: 256 -> 126 + the two flow columns in one N tile of 128; width 100 (one clipped row)
    case("wide_append_flow_126", 2, 9, 100, (3, 3), [(256,)], 126, R.RELU_APPEND_FLOW),
    # two sources, the second at an offset inside a wider stride; one N tile of 96 (Cout 80: the last block is clipped at
    # the layer's last column); 312 items: several per CTA and a partial last round
    case("wide_nt96_two_src", 6, 25, 512, (3, 3), [(128,), (64, 96, 16)], 80, R.RELU),
    # a single row: every item's second row is below the image
    case("wide_single_row", 2, 1, 256, (3, 3), [(192,)], 128, R.RELU),
]
BY_NAME = {c["name"]: c for c in CASES}


@pytest.mark.parametrize("dtype", HALF, ids=["float16", "bfloat16"])
@pytest.mark.parametrize("name", list(BY_NAME))
def test_wide_conformance(name, dtype):
    for impl in (2, 0):  # the wgmma path itself and auto selection
        worst = run(BY_NAME[name], dtype, impl)
        _report(test="conv_wide_conformance", case=name, dtype=str(dtype), impl=impl, max_err_over_bound=worst)


def run_wide_sweep():
    """Every case once per half type (test_cases_take_the_wide_kernel runs this in a subprocess with the launch trace on)."""
    for c in CASES:
        for dt in HALF:
            run(c, dt, 2)


def test_cases_take_the_wide_kernel(tmp_path):
    trace = tmp_path / "conv_trace.jsonl"
    env = dict(os.environ, PFB_CONV_TRACE=str(trace))
    env.pop("PFB_PARITY_REPORT", None)
    code = "import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; import test_gpu_conv_wide as T; T.run_wide_sweep()"
    r = subprocess.run([sys.executable, "-c", code, ROOT, os.path.join(ROOT, "tests")], env=env, cwd=str(tmp_path),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    plans = [json.loads(line) for line in trace.read_text().splitlines() if line.strip()]
    assert len(plans) == 2 * len(CASES)
    for p in plans:
        assert p["wide"] == 1 and (p["TW"], p["TH"], p["halo"]) == (128, 2, 1), {k: v for k, v in p.items() if k != "t"}
    assert {p["NT"] for p in plans} == {96, 128}
    assert {p["epi"] for p in plans} == {R.RELU, R.RELU_APPEND_FLOW}
    assert any(p["n_work"] > 2 * p["grid"] for p in plans)
