"""Write the GMA attention-variant fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of oracle/make_golden.py for GMA's position-only, position-and-content and multi-head
attention.  Usage, from the repository root:

    python tests/make_gma_golden.py

Writes op_gma_variants.npz (Attention / Aggregate of the reference's own gma_utils modules, a seeded sample of each output),
the e2e_gma_* cases of gma_oracle.E2E_CASES and state_shapes_gma_heads4.json.  Inputs and weights are rebuilt from the
recipes by gma_oracle / oracle.synth, so the fixtures hold outputs only.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import gma_oracle as GO  # noqa: E402
from oracle import ref_shim, synth  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")


def _recipe(**kw) -> np.ndarray:
    return np.frombuffer(json.dumps(kw, sort_keys=True).encode(), dtype=np.uint8)


def reference_op_outputs(mode: str, heads: int, b: int, h: int, w: int):
    """The reference's Attention / Aggregate (gma_utils.py:32-113) for one operator case -> (attention, aggregate)."""
    ref_shim.load_gma()
    import ptlflow.models.gma.gma_utils as gu

    sd, inp, motion = GO.op_inputs(heads, b, h, w)
    flags = {"position_only": False, "position_and_content": False, **GO.MODES[mode]}
    att = gu.Attention(dim=128, heads=heads, max_pos_size=160, dim_head=128, **flags).eval()
    agg = gu.Aggregate(dim=128, dim_head=128, heads=heads).eval()
    att.load_state_dict({k[len("att."):]: v for k, v in sd.items() if k.startswith("att.")}, strict=False)  # rel_ind: built in
    agg.load_state_dict({k[len("update_block.aggregator."):]: v for k, v in sd.items() if k.startswith("update_block.")})
    with torch.no_grad():
        a = att(inp)  # [b, heads, N, N]
        g = agg(a, motion)
    return a.numpy().astype(np.float32), g.numpy().astype(np.float32)


def reference_model(seed: int, **kwargs):
    """The reference gma in eval mode holding gma_oracle.synth_state_dict weights."""
    model = ref_shim.load_gma().gma(**kwargs).eval()
    sd = model.state_dict()
    mine = GO.synth_state_dict({k: tuple(v.shape) for k, v in sd.items() if k.split(".")[0] in ("fnet", "cnet", "update_block", "att")}, seed)
    model.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) if k in mine else v for k, v in sd.items()})
    return model


def reference_e2e(recipe):
    model = reference_model(recipe["wseed"], **recipe["kwargs"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    with torch.no_grad():
        return model({"images": img})


def main() -> None:
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    arrays = {}
    for mode, heads, b, h, w in GO.OP_CASES:
        a, g = reference_op_outputs(mode, heads, b, h, w)
        key = f"{mode}_h{heads}_{h}x{w}"
        for name, arr in (("attention", a), ("aggregate", g)):
            flat = arr.reshape(-1)
            arrays[f"{key}_{name}"] = flat[GO.op_sample(flat.size)]
            arrays[f"{key}_{name}_shape"] = np.array(arr.shape, dtype=np.int64)
    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_gma_variants.npz"), recipe=_recipe(seed=GO.OP_SEED, samples=GO.OP_SAMPLES), **arrays)
    for name, kwargs, b, h, w, kind, wseed, iseed in GO.E2E_CASES:
        recipe = dict(variant="gma", kwargs=kwargs, batch=b, height=h, width=w, kind=kind, wseed=wseed, iseed=iseed)
        out = reference_e2e(recipe)
        np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), recipe=_recipe(**recipe),
                            flows=out["flows"].numpy().astype(np.float32), flow_small=out["flow_small"].numpy().astype(np.float32))
        print(name, tuple(out["flows"].shape), "max|flow|", float(out["flows"].abs().max()))
    mm = ref_shim.load_gma().gma(num_heads=4)
    shapes = {k: list(v.shape) for k, v in mm.state_dict().items() if k.split(".")[0] in ("fnet", "cnet", "update_block", "att")}
    with open(os.path.join(GOLDEN_DIR, "state_shapes_gma_heads4.json"), "w") as f:
        json.dump(shapes, f, indent=0)


if __name__ == "__main__":
    main()
