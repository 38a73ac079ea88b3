"""Write the CSFlow fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_flow1d_golden.py for CSFlow.  Usage, from the repository root:

    python tests/make_csflow_golden.py

Writes state_shapes_csflow.json, op_csflow.npz (the strip maps, the initial strip flow, the lookup of the 2-channel pyramid at
seeded coordinates and one update iteration, from the reference's own modules) and the e2e_csflow_* cases of csflow_oracle.E2E_CASES.
Inputs and weights are rebuilt from the recipes by csflow_oracle / oracle.synth, so the fixtures hold outputs only (the warm case also
keeps the first forward's flow_small and the forward-interpolated warm start).

The weight recipe is oracle.synth's with the strip block's BatchNorm weights and biases scaled by csflow_oracle.STRIP_BN_SCALE, so
that the strip maps and the initial flow stay small (main() prints their ranges per case).
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


def load_csflow():
    """-> the reference module ptlflow.models.csflow.csflow."""
    ref_shim.install()
    name = "ptlflow.models.csflow"
    if name not in sys.modules:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "ptlflow", "models", "csflow")]
        sys.modules[name] = m
    import ptlflow.models.csflow.csflow  # noqa: F401

    return sys.modules[name + ".csflow"]


def reference_model(radius: int, seed: int, **kwargs):
    import csflow_oracle as CS

    m = load_csflow().csflow(corr_radius=radius, **kwargs).eval()
    sd = m.state_dict()
    mine = CS.synth_state_dict(radius, seed)
    assert set(mine) == set(sd)
    m.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) for k, v in sd.items()})
    return m


def reference_corr_init(strip_corr_map_w, strip_corr_map_h):
    """csflow.py:177-190, verbatim."""
    corr_w_act = torch.nn.functional.softmax(strip_corr_map_w, dim=3)  # B H1 W1 1 W2
    corr_h_act = torch.nn.functional.softmax(strip_corr_map_h, dim=4)  # B H1 W1 H2 1
    flo_v = corr_w_act.mul(strip_corr_map_w)  # B H1 W1 1 W2
    flo_u = corr_h_act.mul(strip_corr_map_h)  # B H1 W1 H2 1
    flow_v = torch.sum(flo_v, dim=4).squeeze(dim=3)  # B H1 W1
    flow_u = torch.sum(flo_u, dim=3).squeeze(dim=3)  # B H1 W1
    return torch.stack((flow_u, flow_v), dim=1)  # B 2 H1 W1


def reference_ops():
    import csflow_oracle as CS

    mod = load_csflow()
    sd, x = CS.op_inputs()
    m = reference_model(4, CS.OP_SEED)
    f1, f2 = x["f1"], x["f2"]
    with torch.no_grad():
        smap, sw, sh = m.strip_corr_block_v2([f1, f2])
        out = {"sw": sw[:, :, :, 0, :], "sh": sh[:, :, :, :, 0], "corr_init": reference_corr_init(sw, sh)}
        corr_fn = mod.CorrBlock_v2(f1, f2, smap, radius=CS.OP_LOOKUP_RADIUS)
        out[f"lookup_r{CS.OP_LOOKUP_RADIUS}"] = corr_fn(x["coords"])
        net, mask, delta = m.update_block(x["net"], x["inp"], x["corr"], x["flow"])
        out.update(net=net, mask=mask, delta=delta)
    return {k: CS.np32(v) for k, v in out.items()}


def reference_e2e(recipe, trace: bool = False):
    import csflow_oracle as CS

    kw = dict(recipe["kwargs"])
    m = reference_model(kw.pop("corr_radius", 4), recipe["wseed"], **kw)
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    out, seen = {}, {}
    if trace:  # the strip maps of the (last) forward, for the ranges main() prints
        m.strip_corr_block_v2.register_forward_hook(lambda mod, inp, res: seen.update(sw=res[1], sh=res[2]))
    with torch.no_grad():
        if recipe["warm"]:
            from ptlflow.utils.utils import forward_interpolate_batch

            first = m({"images": img})
            out["prev_flow_small"] = CS.np32(first["flow_small"])
            out["flow_init"] = CS.np32(forward_interpolate_batch(first["flow_small"]))
            res = m({"images": img, "prev_preds": {"flow_small": first["flow_small"]}})
        else:
            res = m({"images": img})
    out["flows"] = CS.np32(res["flows"])
    out["flow_small"] = CS.np32(res["flow_small"])
    return (out, seen) if trace else out


def main() -> None:
    if not ref_shim.available():
        raise SystemExit("the reference checkout is not available")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    sd = load_csflow().csflow().state_dict()
    with open(os.path.join(GOLDEN_DIR, "state_shapes_csflow.json"), "w") as f:
        json.dump({k: list(v.shape) for k, v in sd.items()}, f, indent=0)
    import csflow_oracle as CS

    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_csflow.npz"), recipe=_recipe(seed=CS.OP_SEED), **reference_ops())
    for case in CS.E2E_CASES:
        rec = CS.recipe_of(case)
        out, seen = reference_e2e(rec, trace=True)
        np.savez_compressed(os.path.join(GOLDEN_DIR, case[0] + ".npz"), recipe=_recipe(**rec), **out)
        sw, sh = seen["sw"], seen["sh"]
        init = reference_corr_init(sw, sh)
        print(case[0], {k: v.shape for k, v in out.items()}, "max|flow| %.2f" % float(np.abs(out["flows"]).max()),
              "sw [%.4f, %.4f] sh [%.4f, %.4f] initial flow x [%.3f, %.3f] y [%.3f, %.3f] cells" % (
                  sw.min(), sw.max(), sh.min(), sh.max(), init[:, 0].min(), init[:, 0].max(), init[:, 1].min(), init[:, 1].max()))


if __name__ == "__main__":
    main()
