"""Write the LCV fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_csflow_golden.py for LCV.  Usage, from the repository root:

    python tests/make_lcv_golden.py

Writes state_shapes_lcv_raft.json, state_shapes_lcv_raft_small.json, op_lcv.npz (W, the level sizes of a frozen pyramid and its
lookup at seeded coordinates, from the reference's LearnableCorrBlock) and the e2e_lcv_* cases of lcv_oracle.E2E_CASES.  Inputs and
weights are rebuilt from the recipes by lcv_oracle / oracle.synth, so the fixtures hold outputs only (the warm case also keeps the first
forward's flow_small and the forward-interpolated warm start).  The recipes perturb raw_P and raw_D away from the reference's
initialisation, where W = I (lcv_oracle.P_SCALE, D_SCALE).
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import lcv_oracle as LO  # noqa: E402
from oracle import fixtures as F  # noqa: E402


def load_lcv():
    """-> the reference package ptlflow.models.lcv with lcv_raft and corr_lcv imported."""
    return F.load_package("lcv", "lcv_raft", "corr_lcv")


def reference_model(recipe):
    kw = dict(recipe["kwargs"])
    kw.pop("iters", None)
    cls = getattr(load_lcv().lcv_raft, recipe["model"])
    m = cls(iters=recipe["kwargs"].get("iters", 32), **kw)
    m.dtype, m.device = torch.float32, torch.device("cpu")  # what lightning's module gives coords_grid (lcv_raft.py:89-96)
    return F.reference_model(m, lambda _: LO.synth_state_dict(recipe["model"], recipe["wseed"], kw.get("corr_levels", 4),
                                                              kw.get("corr_radius")))


def reference_ops():
    block_cls = load_lcv().corr_lcv.LearnableCorrBlock
    form, f1, f2, coords = LO.op_inputs()
    blk = block_cls(LO.OP_DIM, LO.OP_LEVELS, LO.OP_RADIUS)
    blk.load_state_dict(form)
    with torch.no_grad():
        pyr = blk.compute_cost_volume(f1, f2)
        out = {"W": blk.W, "level_sizes": torch.tensor([tuple(p.shape[-2:]) for p in pyr[:LO.OP_LEVELS]], dtype=torch.float32),
               "lookup": blk(pyr, coords)}
    return {k: F.np32(v) for k, v in out.items()}


def reference_e2e(recipe):
    return F.reference_e2e(reference_model(recipe), recipe)


def main() -> None:
    F.start()
    lcv = load_lcv().lcv_raft
    F.write_state_shapes("lcv_raft", lcv.lcv_raft())
    F.write_state_shapes("lcv_raft_small", lcv.lcv_raft_small())
    F.write_fixture("op_lcv", dict(seed=LO.OP_SEED), reference_ops())
    F.write_e2e(LO.E2E_CASES, LO.recipe_of, reference_model)


if __name__ == "__main__":
    main()
