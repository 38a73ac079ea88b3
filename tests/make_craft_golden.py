"""Write the CRAFT fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_llaflow_golden.py for CRAFT.  Usage, from the repository root:

    python tests/make_craft_golden.py

Writes state_shapes_craft.json and the e2e_craft_* cases of craft_oracle.E2E_CASES.  Inputs and weights are rebuilt from the recipes
by craft_oracle / oracle.synth, so the fixtures hold outputs only (the warm case also keeps the first forward's flow_small and the
forward-interpolated warm start), plus, per case, the largest inter-frame score of each sample (``max_score``).

The reference's constructor reads ``pos_bias_radius`` from ``self.__dict__["_hparams"]`` (craft.py:120), which the training framework
fills from the constructor's arguments; the shared shim's ``save_hyperparameters`` does nothing, so ``reference_class`` supplies them.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import craft_oracle as CR  # noqa: E402
from oracle import fixtures as F  # noqa: E402


def load_craft():
    """-> the reference package ptlflow.models.craft (its modules craft, setrans)."""
    return F.load_package("craft", "craft", "setrans")


def reference_class():
    """The reference's ``craft`` with its hyper-parameters in ``_hparams``, as the training framework would store them."""
    base = load_craft().craft.craft

    class craft_with_hparams(base):
        def __init__(self, **kw):
            self.__dict__["_hparams"] = dict(kw, pos_bias_radius=kw.get("pos_bias_radius", 7))
            super().__init__(**kw)

    return craft_with_hparams


def reference_model(recipe):
    kw = dict(recipe["kwargs"])
    return F.reference_model(reference_class()(**kw), lambda _: CR.synth_state_dict(kw, recipe["wseed"], recipe.get("qscale", 1.0)))


def reference_e2e(recipe):
    return F.reference_e2e(reference_model(recipe), recipe)


def score_maxima(recipe, m):
    """Records the largest inter-frame score of each sample of the (last) forward, before the clamp."""
    seen = {}
    st = getattr(m.corr_fn, "setrans", None) if recipe["kwargs"].get("craft", True) else None
    if st is not None:
        def hook(mod, inp, res):
            x1, x2 = inp[0], inp[1]
            seen["max"] = CR.mode_scores(x1, x2, {k: v for k, v in [("p.query.weight", mod.query.weight), ("p.query.bias", mod.query.bias),
                                                                  ("p.key.weight", mod.key.weight), ("p.key.bias", mod.key.bias)]
                                                  if v is not None}, "p.", mod.num_modes).amax(dim=(1, 2, 3))
        st.register_forward_hook(hook)

    def finish(out):
        if "max" not in seen:
            return ""
        out["max_score"] = F.np32(seen["max"])
        return "max inter-frame score per sample " + ", ".join("%.1f" % v for v in out["max_score"])

    return finish


def main() -> None:
    F.start()
    F.write_state_shapes("craft", reference_class()())
    F.write_e2e(CR.E2E_CASES, CR.recipe_of, reference_model, score_maxima)


if __name__ == "__main__":
    main()
