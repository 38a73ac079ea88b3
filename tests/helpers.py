"""Shared helpers for the parity tests: golden loading and synthetic tensors."""
import json
import os

import numpy as np
import torch

from oracle import raft_oracle as O
from oracle import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    recipe = json.loads(bytes(z["recipe"]).decode())
    return recipe, {k: z[k] for k in z.files if k != "recipe"}


def e2e_inputs(recipe):
    """(state_dict, images, kwargs) rebuilt from a golden recipe (see oracle/make_golden.py)."""
    kw = dict(recipe["kwargs"])
    shapes = O.state_dict_shapes(recipe["variant"], kw.get("corr_levels", 4), kw.get("corr_radius"))
    sd = synth.synth_state_dict(shapes, recipe["wseed"])
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    return sd, img, kw


E2E = ["e2e_raft_small_cfg1", "e2e_raft_small_b2", "e2e_raft_noise", "e2e_raft_smooth_b2", "e2e_raft_altcorr", "e2e_raft_r3_l3", "e2e_gma"]


def load_golden_arrays(name):
    """A golden file without a recipe: every array it holds."""
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: z[k] for k in z.files}


def lib():
    """The ctypes binding (ptlflow_b200._lib), with the library built first where it is missing."""
    from ptlflow_b200 import _lib as L
    from ptlflow_b200.csrc import build as B

    if not os.path.exists(L.LIB_PATH):
        B.build()
    return L


def raft_cfg(L, defaults, **overrides):
    """A pfb_raft_cfg of the fields in ``defaults``, then ``overrides``, by field name; every other field 0."""
    return L.RaftCfg(**{**defaults, **overrides})
