"""Write the SKFlow fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of oracle/make_golden.py for SKFlow.  Usage, from the repository root:

    python tests/make_skflow_golden.py

Writes op_skflow.npz (each PCBlock shape of the default model and one update-block iteration of the reference's own
skflow/update.py modules, a seeded sample of each output), the e2e_skflow_* cases of skflow_oracle.E2E_CASES and
state_shapes_skflow.json.  Inputs and weights are rebuilt from the recipes by skflow_oracle / oracle.synth, so the fixtures hold
outputs only.  The reference package is loaded through oracle/ref_shim plus two additions made here: the skflow namespace package
and the ``dtype`` / ``device`` properties that skflow.py reads from its LightningModule base.
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

import skflow_oracle as SO  # noqa: E402
from oracle import ref_shim, synth  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")


def _recipe(**kw) -> np.ndarray:
    return np.frombuffer(json.dumps(kw, sort_keys=True).encode(), dtype=np.uint8)


def load_skflow():
    """-> the reference module ptlflow.models.skflow.skflow."""
    ref_shim.install()
    name = "ptlflow.models.skflow"
    if name not in sys.modules:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "ptlflow", "models", "skflow")]
        sys.modules[name] = m
    lm = sys.modules["lightning.pytorch"].LightningModule
    if "dtype" not in lm.__dict__:
        lm.dtype = property(lambda self: next(self.parameters()).dtype)
        lm.device = property(lambda self: next(self.parameters()).device)
    import ptlflow.models.skflow.skflow as ref_skflow

    return ref_skflow


def reference_block(name: str, cin: int, cout: int, kind: str, b: int, h: int, w: int) -> np.ndarray:
    load_skflow()
    import ptlflow.models.skflow.update as up

    sd, ks, x = SO.op_block_inputs(name, cin, cout, kind, b, h, w)
    blk = up.PCBlock4_Deep_nopool_res(cin, cout, k_conv=ks).eval()
    blk.load_state_dict(sd)
    with torch.no_grad():
        return blk(x).numpy().astype(np.float32)


def reference_iteration(b: int, h: int, w: int):
    """One SKUpdateBlock6_Deep_nopoolres_AllDecoder evaluation (two heads) -> (net, mask, delta)."""
    load_skflow()
    import ptlflow.models.skflow.update as up

    sd, net, inp, corr, flow, attn = SO.op_iter_inputs(b, h, w)
    blk = up.SKUpdateBlock6_Deep_nopoolres_AllDecoder(4, 4, (1, 15), (1, 7), num_heads=2, hidden_dim=128).eval()
    blk.load_state_dict({k[len("update_block."):]: v for k, v in sd.items() if k.startswith("update_block.")})
    with torch.no_grad():
        n, m, d = blk(net, inp, corr, flow, attn)
    return n.numpy().astype(np.float32), m.numpy().astype(np.float32), d.numpy().astype(np.float32)


def reference_model(seed: int, **kwargs):
    """The reference skflow in eval mode holding skflow_oracle.synth_state_dict weights."""
    model = load_skflow().skflow(**kwargs).eval()
    sd = model.state_dict()
    mine = SO.synth_state_dict({k: tuple(v.shape) for k, v in sd.items() if k.split(".")[0] in ("fnet", "cnet", "update_block", "att")}, seed)
    model.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) if k in mine else v for k, v in sd.items()})
    return model


def reference_e2e(recipe, warm: bool = False):
    """-> (output, first output or None); with ``warm`` the second forward starts from the first one's flow_small."""
    model = reference_model(recipe["wseed"], **recipe["kwargs"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    with torch.no_grad():
        out = model({"images": img})
        if not warm:
            return out, None
        return model({"images": img, "prev_preds": {"flow_small": out["flow_small"]}}), out


def main() -> None:
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    arrays = {}
    for b, h, w in SO.OP_GRIDS:
        for name, cin, cout, kind in SO.OP_BLOCKS:
            out = reference_block(name, cin, cout, kind, b, h, w).reshape(-1)
            arrays[f"{name}_{h}x{w}"] = out[SO.op_sample(out.size)]
        for key, arr in zip(("net", "mask", "delta"), reference_iteration(b, h, w)):
            flat = arr.reshape(-1)
            arrays[f"iter_{key}_{h}x{w}"] = flat[SO.op_sample(flat.size)]
    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_skflow.npz"), recipe=_recipe(seed=SO.OP_SEED, samples=SO.OP_SAMPLES), **arrays)
    for name, kwargs, b, h, w, kind, wseed, iseed, warm in SO.E2E_CASES:
        recipe = dict(variant="skflow", kwargs=kwargs, batch=b, height=h, width=w, kind=kind, wseed=wseed, iseed=iseed, warm=warm)
        out, first = reference_e2e(recipe, warm)
        extra = {} if first is None else {"first_flow_small": first["flow_small"].numpy().astype(np.float32)}
        np.savez_compressed(os.path.join(GOLDEN_DIR, name + ".npz"), recipe=_recipe(**recipe),
                            flows=out["flows"].numpy().astype(np.float32), flow_small=out["flow_small"].numpy().astype(np.float32), **extra)
        print(name, tuple(out["flows"].shape), "max|flow|", float(out["flows"].abs().max()))
    mm = load_skflow().skflow()
    shapes = {k: list(v.shape) for k, v in mm.state_dict().items() if k.split(".")[0] in ("fnet", "cnet", "update_block", "att")}
    with open(os.path.join(GOLDEN_DIR, "state_shapes_skflow.json"), "w") as f:
        json.dump(shapes, f, indent=0)


if __name__ == "__main__":
    main()
