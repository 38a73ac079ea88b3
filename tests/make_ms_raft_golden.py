"""Write the MS-RAFT+ fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_sea_raft_golden.py for MS-RAFT+.  Usage, from the repository root:

    python tests/make_ms_raft_golden.py

Writes op_ms_raft_p.npz (a stride-2 group-norm residual block, an up layer, one update iteration's net / delta / mask and both convex
2x modes, from the reference's own modules and functions), the e2e_ms_raft_p_* cases of ms_raft_oracle.E2E_CASES and
state_shapes_ms_raft_p.json.  Inputs and weights are rebuilt from the recipes by ms_raft_oracle / oracle.synth, so the fixtures hold
outputs only (the warm case also keeps the first forward's flow_small and the reference's forward-interpolated warm start).  The
reference package is loaded through oracle/ref_shim plus the ms_raft_plus namespace package; without the compiled alt_cuda_corr
plugin its alternate_corr=True path runs IterativeCorrBlock.
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import ms_raft_oracle as MS  # noqa: E402
from oracle import ref_shim, synth  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")


def _recipe(**kw) -> np.ndarray:
    return np.frombuffer(json.dumps(kw, sort_keys=True).encode(), dtype=np.uint8)


def load_ms_raft():
    """-> the reference module ptlflow.models.ms_raft_plus.ms_raft_plus."""
    ref_shim.install()
    name = "ptlflow.models.ms_raft_plus"
    if name not in sys.modules:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "ptlflow", "models", "ms_raft_plus")]
        sys.modules[name] = m
    import ptlflow.models.ms_raft_plus.ms_raft_plus as ref

    return ref


def reference_model(seed: int, **kwargs):
    """The reference ms_raft_p in eval mode holding ms_raft_oracle.synth_state_dict weights."""
    model = load_ms_raft().ms_raft_p(**kwargs).eval()
    sd = model.state_dict()
    mine = MS.synth_state_dict({k: tuple(v.shape) for k, v in sd.items()}, seed)
    model.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) for k, v in sd.items()})
    return model


def reference_ops():
    sd, x = MS.op_inputs()
    model = load_ms_raft().ms_raft_p().eval()
    model.load_state_dict({k: v.to(model.state_dict()[k].dtype) for k, v in sd.items()})
    f = model.fnet
    import torchvision.transforms.functional as TF

    with torch.no_grad():
        block = f.layer2[0](x["block_in"])
        up = x["up_skip"]
        up = f.up_layer1(torch.cat([TF.resize(x["up_coarse"], list(up.shape[-2:])), up], 1))
        net, mask, delta = model.update_block(x["net"], x["inp"], x["corr"], x["flow"])
        grid = MS.O.coords_grid(2, 6, 9)
        up_flow = model.upsample_flow(x["coords"] - grid, x["mask"], scale=2)
        up_coords = model.upsample_flow(x["coords"], x["mask"], scale=2)
    return {k: MS.np32(v) for k, v in dict(block=block, up_layer=up, net=net, mask=mask, delta=delta, up_flow=up_flow,
                                           up_coords=up_coords).items()}


def reference_e2e(recipe):
    model = reference_model(recipe["wseed"], **recipe["kwargs"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    out = {}
    with torch.no_grad():
        if recipe["warm"]:
            from ptlflow.utils.utils import forward_interpolate_batch

            first = model({"images": img})
            out["prev_flow_small"] = MS.np32(first["flow_small"])
            out["flow_init"] = MS.np32(forward_interpolate_batch(first["flow_small"]))
            res = model({"images": img, "prev_preds": {"flow_small": first["flow_small"]}})
        else:
            res = model({"images": img})
    out["flows"] = MS.np32(res["flows"])
    out["flow_small"] = MS.np32(res["flow_small"])
    return out


def main() -> None:
    if not ref_shim.available():
        raise SystemExit("the reference checkout is not available")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_ms_raft_p.npz"), recipe=_recipe(seed=MS.OP_SEED), **reference_ops())
    for case in MS.E2E_CASES:
        rec = MS.recipe_of(case)
        out = reference_e2e(rec)
        np.savez_compressed(os.path.join(GOLDEN_DIR, case[0] + ".npz"), recipe=_recipe(**rec), **out)
        print(case[0], {k: v.shape for k, v in out.items()}, "max|flow| %.1f" % float(np.abs(out["flows"]).max()))
    sd = reference_model(0).state_dict()
    with open(os.path.join(GOLDEN_DIR, "state_shapes_ms_raft_p.json"), "w") as f:
        json.dump({k: list(v.shape) for k, v in sd.items()}, f, indent=0)


if __name__ == "__main__":
    main()
