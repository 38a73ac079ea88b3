"""CPU: the timing presets expand to the runs and kernel cases they promise, and the event timer refuses to run without a
CUDA device instead of timing something else."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

import time_kernels  # noqa: E402
import time_models  # noqa: E402
import timing  # noqa: E402

S, K4 = "1024x436", "3840x2160"


EXPECTED = {  # preset: (runs in the order they are timed, runs that add an eager forward's fields, kernel cases)
    "gma_variants": (
        [("gma", {}, "bf16", 4, 12, S), ("gma", {"position_only": True}, "bf16", 4, 12, S),
         ("gma", {"position_and_content": True}, "bf16", 4, 12, S), ("gma", {"num_heads": 4}, "bf16", 4, 12, S)],
        [], ["attention_softmax_relpos"]),
    "skflow": (
        [("skflow", {}, "bf16", 4, 12, S), ("skflow", {}, "bf16", 8, 12, S), ("skflow", {}, "f16", 4, 12, S), ("skflow", {}, "f16", 8, 12, S)],
        "all", ["depthwise_conv_gelu"]),
    "sea_raft": (
        [("sea_raft_s", {}, "bf16", 4, None, S), ("sea_raft_s", {}, "bf16", 8, None, S), ("sea_raft_s", {}, "f16", 4, None, S),
         ("sea_raft_s", {}, "f16", 8, None, S), ("sea_raft_l", {}, "bf16", 4, None, S), ("sea_raft_l", {}, "bf16", 8, None, S),
         ("sea_raft_l", {}, "f16", 4, None, S), ("sea_raft_l", {}, "f16", 8, None, S)],
        "all", ["depthwise_conv_layernorm"]),
    "ms_raft": (
        [("ms_raft_p", {}, "bf16", 1, None, S), ("ms_raft_p", {}, "bf16", 2, None, S), ("ms_raft_p", {}, "bf16", 4, None, S),
         ("ms_raft_p", {}, "f16", 1, None, S), ("ms_raft_p", {}, "f16", 2, None, S), ("ms_raft_p", {}, "f16", 4, None, S)],
        [("ms_raft_p", {}, "bf16", 1, None, S)], []),
    "ccmr": (
        [("ccmr", {}, "bf16", 1, None, S), ("ccmr", {}, "bf16", 2, None, S), ("ccmr", {}, "f16", 1, None, S), ("ccmr", {}, "f16", 2, None, S),
         ("ccmr_p", {}, "bf16", 1, None, S), ("ccmr_p", {}, "bf16", 2, None, S), ("ccmr_p", {}, "f16", 1, None, S),
         ("ccmr_p", {}, "f16", 2, None, S)],
        [("ccmr", {}, "bf16", 1, None, S), ("ccmr_p", {}, "bf16", 1, None, S)], []),
    "flow1d": (
        [("flow1d", {}, "bf16", 1, 12, S), ("flow1d", {}, "bf16", 1, 32, S), ("flow1d", {}, "bf16", 4, 12, S), ("flow1d", {}, "bf16", 4, 32, S),
         ("flow1d", {}, "bf16", 1, 12, K4), ("flow1d", {}, "bf16", 1, 32, K4),
         ("flow1d", {}, "f16", 1, 12, S), ("flow1d", {}, "f16", 1, 32, S), ("flow1d", {}, "f16", 4, 12, S), ("flow1d", {}, "f16", 4, 32, S)],
        [("flow1d", {}, "bf16", 1, 32, S)], ["attn1d", "corr1d_lookup"]),
    "csflow": (
        [("csflow", {}, "bf16", 1, 12, S), ("csflow", {}, "bf16", 1, 32, S), ("csflow", {}, "bf16", 4, 12, S), ("csflow", {}, "bf16", 4, 32, S),
         ("csflow", {}, "f16", 1, 12, S), ("csflow", {}, "f16", 1, 32, S), ("csflow", {}, "f16", 4, 12, S), ("csflow", {}, "f16", 4, 32, S),
         ("raft", {}, "bf16", 1, 12, S), ("raft", {}, "bf16", 1, 32, S), ("raft", {}, "bf16", 4, 12, S), ("raft", {}, "bf16", 4, 32, S),
         ("raft", {}, "f16", 1, 12, S), ("raft", {}, "f16", 1, 32, S), ("raft", {}, "f16", 4, 12, S), ("raft", {}, "f16", 4, 32, S)],
        [("csflow", {}, "bf16", 1, 32, S), ("raft", {}, "bf16", 1, 32, S)], []),
    "scv": (
        [("scv4", {}, "bf16", 1, 12, S), ("scv4", {}, "bf16", 1, 32, S), ("scv4", {}, "bf16", 4, 12, S), ("scv4", {}, "bf16", 4, 32, S),
         ("scv4", {}, "f16", 1, 12, S), ("scv4", {}, "f16", 1, 32, S), ("scv4", {}, "f16", 4, 12, S), ("scv4", {}, "f16", 4, 32, S),
         ("scv8", {}, "bf16", 1, 12, S), ("scv8", {}, "bf16", 1, 32, S), ("scv8", {}, "bf16", 4, 12, S), ("scv8", {}, "bf16", 4, 32, S),
         ("scv8", {}, "f16", 1, 12, S), ("scv8", {}, "f16", 1, 32, S), ("scv8", {}, "f16", 4, 12, S), ("scv8", {}, "f16", 4, 32, S),
         ("raft", {}, "bf16", 1, 12, S), ("raft", {}, "bf16", 1, 32, S), ("raft", {}, "bf16", 4, 12, S), ("raft", {}, "bf16", 4, 32, S),
         ("raft", {}, "f16", 1, 12, S), ("raft", {}, "f16", 1, 32, S), ("raft", {}, "f16", 4, 12, S), ("raft", {}, "f16", 4, 32, S)],
        [("scv4", {}, "bf16", 1, 32, S)], ["knn_topk", "sparse_lookup"]),
    "llaflow": (
        [("llaflow", {}, "bf16", 1, 12, S), ("llaflow", {}, "bf16", 1, 32, S), ("llaflow", {}, "bf16", 4, 12, S), ("llaflow", {}, "bf16", 4, 32, S),
         ("llaflow", {}, "f16", 1, 12, S), ("llaflow", {}, "f16", 1, 32, S), ("llaflow", {}, "f16", 4, 12, S), ("llaflow", {}, "f16", 4, 32, S),
         ("llaflow_raft", {}, "bf16", 1, 12, S), ("llaflow_raft", {}, "bf16", 1, 32, S), ("llaflow_raft", {}, "bf16", 4, 12, S),
         ("llaflow_raft", {}, "bf16", 4, 32, S), ("llaflow_raft", {}, "f16", 1, 12, S), ("llaflow_raft", {}, "f16", 1, 32, S),
         ("llaflow_raft", {}, "f16", 4, 12, S), ("llaflow_raft", {}, "f16", 4, 32, S),
         ("gma", {}, "bf16", 1, 12, S), ("gma", {}, "bf16", 1, 32, S), ("gma", {}, "bf16", 4, 12, S), ("gma", {}, "bf16", 4, 32, S),
         ("gma", {}, "f16", 1, 12, S), ("gma", {}, "f16", 1, 32, S), ("gma", {}, "f16", 4, 12, S), ("gma", {}, "f16", 4, 32, S),
         ("raft", {}, "bf16", 1, 12, S), ("raft", {}, "bf16", 1, 32, S), ("raft", {}, "bf16", 4, 12, S), ("raft", {}, "bf16", 4, 32, S),
         ("raft", {}, "f16", 1, 12, S), ("raft", {}, "f16", 1, 32, S), ("raft", {}, "f16", 4, 12, S), ("raft", {}, "f16", 4, 32, S)],
        [], ["shift_volume_tiled"]),
}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_preset_expands_to_its_runs(name):
    runs, eager, kernels = EXPECTED[name]
    preset = time_models.PRESETS[name]
    got = time_models.expand(preset)
    assert [tuple(r) for r in got] == runs
    assert [tuple(r) for r in got if any(time_models.matches(r, fields) for fields, _ in preset.eager)] == (runs if eager == "all" else eager)
    assert list(preset.kernels) == kernels
    assert all(k in time_kernels.CASES for k in kernels)


def test_every_preset_is_checked():
    assert sorted(time_models.PRESETS) == sorted(EXPECTED)


def test_events_ms_needs_a_cuda_device(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA device"):
        timing.events_ms(lambda: None, 1, 0)
