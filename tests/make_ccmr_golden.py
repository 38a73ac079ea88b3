"""Write the CCMR fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_ms_raft_golden.py for CCMR / CCMR+.  Usage, from the repository root:

    python tests/make_ccmr_golden.py

Writes state_shapes_ccmr.json / state_shapes_ccmr_p.json, op_ccmr.npz (an XCiT self-attention block, an aggregator block, one update
iteration, the scale handover and upflow2, from the reference's own modules and functions) and the e2e_ccmr* cases of
ccmr_oracle.E2E_CASES.  Inputs and weights are rebuilt from the recipes by ccmr_oracle / oracle.synth, so the fixtures hold outputs
only (the warm case also keeps the first forward's flow_small and the forward-interpolated warm start).

The reference package is loaded through oracle/ref_shim plus a ``ccmr`` namespace package.  Its xcit.py imports
``timm.models.vision_transformer.Mlp`` and ``timm.models.layers.{DropPath, trunc_normal_, to_2tuple}``; when timm is absent this
script alone installs stand-ins for those names, none of which enters the eval math:
  - ``Mlp`` and ``to_2tuple`` are shadowed by xcit.py's own definitions (``class Mlp`` and ``from .helpers import to_2tuple``);
  - ``DropPath`` (drop_path_rate 0.05) is the identity in eval;
  - ``trunc_normal_`` only initialises weights (``init_weights``, never called by the model), and the fixtures overwrite every weight.
"""
from __future__ import annotations

import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from oracle import ref_shim, synth  # noqa: E402

GOLDEN_DIR = os.path.join(HERE, "golden")


def _recipe(**kw) -> np.ndarray:
    return np.frombuffer(json.dumps(kw, sort_keys=True).encode(), dtype=np.uint8)


def _timm_standins() -> None:
    try:
        import timm  # noqa: F401
        return
    except ImportError:
        pass

    class _DropPath(nn.Identity):
        def __init__(self, *a, **k):
            super().__init__()

    def _trunc_normal_(t, *a, **k):
        return t

    def _unused(*a, **k):
        raise RuntimeError("timm stand-in: shadowed by xcit.py's own definition")

    mods = {n: types.ModuleType(n) for n in ("timm", "timm.models", "timm.models.vision_transformer", "timm.models.layers")}
    mods["timm.models.vision_transformer"].Mlp = _unused
    mods["timm.models.layers"].DropPath = _DropPath
    mods["timm.models.layers"].trunc_normal_ = _trunc_normal_
    mods["timm.models.layers"].to_2tuple = _unused
    sys.modules.update(mods)


def load_ccmr():
    """-> the reference module ptlflow.models.ccmr.ccmr."""
    ref_shim.install()
    _timm_standins()
    name = "ptlflow.models.ccmr"
    if name not in sys.modules:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "ptlflow", "models", "ccmr")]
        sys.modules[name] = m
    import ptlflow.models.ccmr.ccmr as ref

    return ref


def reference_model(model: str, seed: int, **kwargs):
    import ccmr_oracle as CC

    m = getattr(load_ccmr(), model)(**kwargs).eval()
    sd = m.state_dict()
    mine = CC.synth_state_dict({k: tuple(v.shape) for k, v in sd.items()}, seed)
    m.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) for k, v in sd.items()})
    return m


def reference_ops():
    import ccmr_oracle as CC

    sd, x = CC.op_inputs()
    m = load_ccmr().ccmr_p().eval()
    m.load_state_dict({k: v.to(m.state_dict()[k].dtype) for k, v in sd.items()})
    with torch.no_grad():
        gc_self = m.xcit[1](x["ctx"])
        agg = m.update_block.aggregator[1](x["gc"], x["ctx"])
        net, mask, delta = m.update_block(x["net"], x["inp"], x["corr"], x["flow"], x["gc"], level_index=1)
        grid = CC.O.coords_grid(2, 12, 18)
        handover = grid + m.upsample_flow(x["coords"] - CC.O.coords_grid(2, 6, 9), x["mask"], scale=2)
        from ptlflow.models.ccmr.utils import upflow2

        up2 = upflow2(x["flow_lo"])
    return {k: CC.np32(v) for k, v in dict(xcit_self=gc_self, xcit_agg=agg, net=net, mask=mask, delta=delta, handover=handover,
                                            upflow2=up2).items()}


def reference_e2e(recipe):
    import ccmr_oracle as CC

    m = reference_model(recipe["model"], recipe["wseed"], **recipe["kwargs"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    out = {}
    with torch.no_grad():
        if recipe["warm"]:
            from ptlflow.utils.utils import forward_interpolate_batch

            first = m({"images": img})
            out["prev_flow_small"] = CC.np32(first["flow_small"])
            out["flow_init"] = CC.np32(forward_interpolate_batch(first["flow_small"]))
            res = m({"images": img, "prev_preds": {"flow_small": first["flow_small"]}})
        else:
            res = m({"images": img})
    out["flows"] = CC.np32(res["flows"])
    out["flow_small"] = CC.np32(res["flow_small"])
    return out


def main() -> None:
    if not ref_shim.available():
        raise SystemExit("the reference checkout is not available")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    for model in ("ccmr", "ccmr_p"):
        sd = getattr(load_ccmr(), model)().state_dict()
        with open(os.path.join(GOLDEN_DIR, f"state_shapes_{model}.json"), "w") as f:
            json.dump({k: list(v.shape) for k, v in sd.items()}, f, indent=0)
    import ccmr_oracle as CC

    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_ccmr.npz"), recipe=_recipe(seed=CC.OP_SEED), **reference_ops())
    for case in CC.E2E_CASES:
        rec = CC.recipe_of(case)
        out = reference_e2e(rec)
        np.savez_compressed(os.path.join(GOLDEN_DIR, case[0] + ".npz"), recipe=_recipe(**rec), **out)
        print(case[0], {k: v.shape for k, v in out.items()}, "max|flow| %.1f" % float(np.abs(out["flows"]).max()))


if __name__ == "__main__":
    main()
