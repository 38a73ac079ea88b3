"""CPU: the refinement-loop variants.

The pfb_variant enum of include/ptlflow_b200.h against its ctypes mirror, and the workspace of every loop entry point over a fixed
matrix of cfgs against tests/golden/loop_workspace_matrix.npz.  A workspace of 0 bytes is a refusal, so the matrix pins every
decision the loops' cfg checks and workspace plans make.  Re-record it (only for an intended change of those decisions) with
    python tests/test_loop_variants.py --record
"""
import ctypes as C
import itertools
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

from helpers import GOLDEN, lib as _lib  # noqa: E402

MATRIX = os.path.join(GOLDEN, "loop_workspace_matrix.npz")
ENTRY_POINTS = ("pfb_raft_workspace_bytes", "pfb_msraft_workspace_bytes", "pfb_ccmr_workspace_bytes", "pfb_skflow_workspace_bytes",
                "pfb_searaft_workspace_bytes")
# (field(s), values): the Cartesian product of these, in this order, with the last axis varying fastest
AXES = (
    (("variant",), range(-1, 12)),
    (("dtype",), range(4)),
    (("corr_levels",), (1, 4, 5)),
    (("corr_radius",), (0, 3, 4, 16, 64, 65)),
    (("alternate_corr",), (0, 1)),
    (("volume_layout",), (0, 1)),
    (("feat_dim",), (0, 32, 33)),
    (("H", "W"), ((12, 16), (2, 4), (1, 1))),
    (("hidden_dim", "context_dim"), ((128, 128), (96, 64))),
    (("iters",), (0, 1)),
    (("num_heads",), (1, 4)),
)


def workspace_matrix(L) -> np.ndarray:
    """[cfgs, entry points] workspace bytes of every cfg of AXES (B = 2, the output window 8x the grid)."""
    lib = L.load()
    fns = [getattr(lib, name) for name in ENTRY_POINTS]
    cfg = L.RaftCfg(B=2)
    ref = C.byref(cfg)
    rows = []
    for combo in itertools.product(*[values for _, values in AXES]):
        for (fields, _), value in zip(AXES, combo):
            for f, v in zip(fields, value if len(fields) > 1 else (value,)):
                setattr(cfg, f, v)
        cfg.out_h, cfg.out_w = 8 * cfg.H, 8 * cfg.W
        rows.append([fn(ref) for fn in fns])
    return np.array(rows, dtype=np.uint64)


def _axes_record():
    return np.array(repr([(fields, list(values)) for fields, values in AXES]))


def test_variant_enum_equals_lib_constants():
    L = _lib()
    text = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", "ptlflow_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef\s+enum\s*\{([^}]*)\}\s*pfb_variant\s*;", text, flags=re.S).group(1)
    names = [n.split("=")[0].strip() for n in body.split(",") if n.strip()]
    assert names[0] == "PFB_VARIANT_RAFT" and names[-1] == "PFB_VARIANT_COUNT"
    assert re.search(r"PFB_VARIANT_RAFT\s*=\s*0\s*,", body) and body.count("=") == 1  # every value is its position
    for i, n in enumerate(names):
        assert getattr(L, n[len("PFB_"):]) == i, n
    assert sorted(n for n in dir(L) if n.startswith("VARIANT_")) == sorted(n[len("PFB_"):] for n in names)


def test_workspace_matrix_equals_recorded():
    g = np.load(MATRIX)
    assert str(g["axes"]) == str(_axes_record()) and list(g["entry_points"]) == list(ENTRY_POINTS)
    got = workspace_matrix(_lib())
    want = g["bytes"]
    assert got.shape == want.shape
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{len(bad)} entries differ, first (cfg, entry point) {bad[:5].tolist()}: got {got[tuple(bad[0])]}, want {want[tuple(bad[0])]}"
    assert (want.any(axis=1)).sum() > 0  # the recording is not all refusals


if __name__ == "__main__":
    if sys.argv[1:] != ["--record"]:
        sys.exit(__doc__)
    m = workspace_matrix(_lib())
    np.savez_compressed(MATRIX, bytes=m, axes=_axes_record(), entry_points=np.array(ENTRY_POINTS))
    print(f"{MATRIX}: {m.shape[0]} cfgs x {m.shape[1]} entry points, {(m.any(axis=1)).sum()} accepted by at least one")
