"""Write the Flow1D fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_ccmr_golden.py for Flow1D.  Usage, from the repository root:

    python tests/make_flow1d_golden.py

Writes state_shapes_flow1d.json, op_flow1d.npz (the position embedding, both Attention1D directions, both 1D lookups and one update
iteration, from the reference's own modules) and the e2e_flow1d_* cases of flow1d_oracle.E2E_CASES.  Inputs and weights are
rebuilt from the recipes by flow1d_oracle / oracle.synth, so the fixtures hold outputs only (the warm case also keeps the first
forward's flow_small and the forward-interpolated warm start).
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

from oracle import ref_shim, synth  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")


def _recipe(**kw) -> np.ndarray:
    return np.frombuffer(json.dumps(kw, sort_keys=True).encode(), dtype=np.uint8)


def load_flow1d():
    """-> the reference package ptlflow.models.flow1d (its modules flow1d, correlation, position)."""
    ref_shim.install()
    name = "ptlflow.models.flow1d"
    if name not in sys.modules:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "ptlflow", "models", "flow1d")]
        sys.modules[name] = m
    import ptlflow.models.flow1d.correlation  # noqa: F401
    import ptlflow.models.flow1d.flow1d  # noqa: F401
    import ptlflow.models.flow1d.position  # noqa: F401

    return sys.modules[name]


def reference_model(radius: int, seed: int, **kwargs):
    import flow1d_oracle as FD

    m = load_flow1d().flow1d.flow1d(corr_radius=radius, **kwargs).eval()
    sd = m.state_dict()
    mine = FD.synth_state_dict(radius, seed)
    assert set(mine) == set(sd)
    m.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) for k, v in sd.items()})
    return m


def reference_ops():
    import flow1d_oracle as FD

    pkg = load_flow1d()
    sd, x = FD.op_inputs()
    m = reference_model(FD.OP_RADIUS, FD.OP_SEED)
    f1, f2 = x["f1"], x["f2"]
    with torch.no_grad():
        pos = pkg.position.PositionEmbeddingSine(128)(f1)
        f2_x = m.attn_x(f1, f2, pos)[0]
        f2_y = m.attn_y(f1, f2, pos)[0]
        out = {"position": pos[0], "attn_x": f2_x, "attn_y": f2_y}
        for r in (1, FD.OP_RADIUS, 32):
            cx = pkg.correlation.Correlation1D(f1, f2_y, radius=r, x_correlation=True)
            cy = pkg.correlation.Correlation1D(f1, f2_x, radius=r, x_correlation=False)
            out[f"lookup_x_r{r}"], out[f"lookup_y_r{r}"] = cx(x["coords"]), cy(x["coords"])
        net, mask, delta = m.update_block(x["net"], x["inp"], x["corr"], x["flow"], upsample=True)
        out.update(net=net, mask=mask, delta=delta)
    return {k: FD.np32(v) for k, v in out.items()}


def reference_e2e(recipe):
    import flow1d_oracle as FD

    kw = dict(recipe["kwargs"])
    m = reference_model(kw.pop("corr_radius", 32), recipe["wseed"], **kw)
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    out = {}
    with torch.no_grad():
        if recipe["warm"]:
            from ptlflow.utils.utils import forward_interpolate_batch

            first = m({"images": img})
            out["prev_flow_small"] = FD.np32(first["flow_small"])
            out["flow_init"] = FD.np32(forward_interpolate_batch(first["flow_small"]))
            res = m({"images": img, "prev_preds": {"flow_small": first["flow_small"]}})
        else:
            res = m({"images": img})
    out["flows"] = FD.np32(res["flows"])
    out["flow_small"] = FD.np32(res["flow_small"])
    return out


def main() -> None:
    if not ref_shim.available():
        raise SystemExit("the reference checkout is not available")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    sd = load_flow1d().flow1d.flow1d().state_dict()
    with open(os.path.join(GOLDEN_DIR, "state_shapes_flow1d.json"), "w") as f:
        json.dump({k: list(v.shape) for k, v in sd.items()}, f, indent=0)
    import flow1d_oracle as FD

    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_flow1d.npz"), recipe=_recipe(seed=FD.OP_SEED), **reference_ops())
    for case in FD.E2E_CASES:
        rec = FD.recipe_of(case)
        out = reference_e2e(rec)
        np.savez_compressed(os.path.join(GOLDEN_DIR, case[0] + ".npz"), recipe=_recipe(**rec), **out)
        print(case[0], {k: v.shape for k, v in out.items()}, "max|flow| %.1f" % float(np.abs(out["flows"]).max()))


if __name__ == "__main__":
    main()
