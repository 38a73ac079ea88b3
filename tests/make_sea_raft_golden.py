"""Write the SEA-RAFT fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_skflow_golden.py for SEA-RAFT.  Usage, from the repository root:

    python tests/make_sea_raft_golden.py

Writes op_sea_raft.npz (one ConvNextBlock and one update iteration's net / delta / mask of the reference's own modules, a seeded
sample of each output, on two grids), the e2e_sea_raft_* cases of sea_raft_oracle.E2E_CASES and state_shapes_sea_raft*.json.
Inputs and weights are rebuilt from the recipes by sea_raft_oracle / oracle.synth, so the fixtures hold outputs only.  The
reference package is loaded through oracle/ref_shim plus the sea_raft namespace package.  ``block_dims`` is passed as a list:
the reference scales it in place, which its own tuple default does not allow.
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

import sea_raft_oracle as SR  # noqa: E402
from oracle import ref_shim, synth  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")


def _recipe(**kw) -> np.ndarray:
    return np.frombuffer(json.dumps(kw, sort_keys=True).encode(), dtype=np.uint8)


def load_sea_raft():
    """-> the reference module ptlflow.models.sea_raft.sea_raft."""
    ref_shim.install()
    name = "ptlflow.models.sea_raft"
    if name not in sys.modules:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "ptlflow", "models", "sea_raft")]
        sys.modules[name] = m
    import ptlflow.models.sea_raft.sea_raft as ref

    return ref


def reference_model(name: str, seed: int, **kwargs):
    """The registered reference model ``name`` in eval mode holding sea_raft_oracle.synth_state_dict weights."""
    model = getattr(load_sea_raft(), name)(block_dims=[64, 128, 256], **kwargs).eval()
    sd = model.state_dict()
    mine = SR.synth_state_dict({k: tuple(v.shape) for k, v in sd.items()}, seed)
    model.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) for k, v in sd.items()})
    return model


def reference_ops(b: int, h: int, w: int):
    """-> (ConvNextBlock output, net, delta, mask) of the reference's own modules on the op_sea_raft inputs."""
    sd, net, inp, corr, flow = SR.op_inputs(b, h, w)
    model = getattr(load_sea_raft(), "sea_raft")(block_dims=[64, 128, 256], iters=1).eval()
    model.load_state_dict({k: v.to(model.state_dict()[k].dtype) for k, v in sd.items()})
    with torch.no_grad():
        x = torch.cat([net, inp, corr[:, :126], flow], 1)
        blk = model.update_block.refine[0](x)
        n = model.update_block(net, inp, corr, flow)
        d = model.flow_head(n)[:, :2]
        m = 0.25 * model.upsample_weight(n)
    return [t.numpy().astype(np.float32) for t in (blk, n, d, m)]


def reference_e2e(recipe):
    model = reference_model(recipe["model"], recipe["wseed"], **recipe["kwargs"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    with torch.no_grad():
        return model({"images": img})


def main() -> None:
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    arrays = {}
    for b, h, w in SR.OP_GRIDS:
        for key, arr in zip(("block", "net", "delta", "mask"), reference_ops(b, h, w)):
            flat = arr.reshape(-1)
            arrays[f"{key}_{h}x{w}"] = flat[SR.op_sample(flat.size)]
    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_sea_raft.npz"), recipe=_recipe(seed=SR.OP_SEED, samples=SR.OP_SAMPLES), **arrays)
    for name, model, kwargs, b, h, w, kind, wseed, iseed in SR.E2E_CASES:
        recipe = dict(model=model, kwargs=kwargs, batch=b, height=h, width=w, kind=kind, wseed=wseed, iseed=iseed)
        out = reference_e2e(recipe)
        np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), recipe=_recipe(**recipe),
                            flows=out["flows"].numpy().astype(np.float32), flow_small=out["flow_small"].numpy().astype(np.float32))
        print(name, tuple(out["flows"].shape), "max|flow|", float(out["flows"].abs().max()))
    for fname, model, kw in (("state_shapes_sea_raft.json", "sea_raft", {}), ("state_shapes_sea_raft_m.json", "sea_raft_m", {}),
                             ("state_shapes_sea_raft_iters0.json", "sea_raft", {"iters": 0})):
        m = getattr(load_sea_raft(), model)(block_dims=[64, 128, 256], **kw)
        with open(os.path.join(GOLDEN_DIR, fname), "w") as f:
            json.dump({k: list(v.shape) for k, v in m.state_dict().items()}, f, indent=0)


if __name__ == "__main__":
    main()
