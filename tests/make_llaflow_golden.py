"""Write the LLA-Flow fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of tests/make_csflow_golden.py for LLA-Flow.  Usage, from the repository root:

    python tests/make_llaflow_golden.py

Writes state_shapes_llaflow.json, state_shapes_llaflow_raft.json, op_llaflow.npz (both attention tables, fmap2', the volume at
seeded features, borders included, and one GMA update iteration, from the reference's own modules) and the e2e_llaflow_* cases of
llaflow_oracle.E2E_CASES.  Inputs and weights are rebuilt from the recipes by llaflow_oracle / oracle.synth, so the fixtures hold
outputs only (the warm cases also keep the first forward's flow_small and the forward-interpolated warm start).

The weights are oracle.synth's, whose scalar gammas are 0.5 + 0.1 N(0, 1): the volume's gamma and lsa.gamma, both 0 at the
reference's initialisation, are non-zero in every fixture.  main() prints, per case, the max-abs of the gamma corr2 term over that of
the plain term.
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


def load_llaflow():
    """-> the reference module ptlflow.models.llaflow.llaflow."""
    ref_shim.install()
    name = "ptlflow.models.llaflow"
    if name not in sys.modules:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(ref_shim.REFERENCE_ROOT, "ptlflow", "models", "llaflow")]
        sys.modules[name] = m
    import ptlflow.models.llaflow.llaflow  # noqa: F401

    return sys.modules[name + ".llaflow"]


def reference_model(model: str, radius: int, seed: int, **kwargs):
    import llaflow_oracle as LL

    m = getattr(load_llaflow(), model)(corr_radius=radius, **kwargs).eval()
    sd = m.state_dict()
    mine = LL.synth_state_dict(model, radius, seed)
    assert set(mine) == set(sd)
    m.load_state_dict({k: mine[k].to(v.dtype).reshape(v.shape) for k, v in sd.items()})
    return m


def reference_volume(m, fmap1, fmap2, inp):
    """(a1, a2, fmap2', plain term, gamma corr2) of llaflow.py:167-177 and corr.py:13-14, from the reference's own modules."""
    mod = sys.modules["ptlflow.models.llaflow.corr"]
    ls1, ls2 = m.ls1(inp), m.ls2(inp)
    fmap2p = m.lsa(ls2, fmap2)
    corr2 = m.s_lsa(ls1, fmap1, fmap2p)
    plain = mod.CorrBlock.corr(fmap1, fmap2p)
    b, h, w = fmap1.shape[0], fmap1.shape[2], fmap1.shape[3]
    return ls1[:, 0], ls2[:, 0], fmap2p, plain.reshape(b * h * w, 1, h, w), (m.gamma * corr2).reshape(b * h * w, 1, h, w)


def reference_ops():
    import llaflow_oracle as LL

    sd, x = LL.op_inputs()
    m = reference_model("llaflow", 4, LL.OP_SEED)
    with torch.no_grad():
        a1, a2, fmap2p, plain, extra = reference_volume(m, x["fmap1"], x["fmap2"], x["inp"])
        full = load_llaflow().CorrBlock(x["fmap1"], fmap2p, m.gamma, m.s_lsa(m.ls1(x["inp"]), x["fmap1"], fmap2p))
        out = {"a1": a1, "a2": a2, "fmap2p": fmap2p, "volume": full.corr_pyramid[0]}
        assert torch.allclose(full.corr_pyramid[0], plain + extra, atol=1e-6, rtol=0)
        attn = m.att(x["it_inp"])
        net, mask, delta = m.update_block(x["it_net"], x["it_inp"], x["it_corr"], x["it_flow"], attn)
        out.update(net=net, mask=mask, delta=delta)
    return {k: LL.np32(v) for k, v in out.items()}


def reference_e2e(recipe, trace: bool = False):
    import llaflow_oracle as LL

    kw = dict(recipe["kwargs"])
    m = reference_model(recipe["model"], kw.pop("corr_radius", 4), recipe["wseed"], **kw)
    img = torch.from_numpy(synth.synth_images(recipe["batch"], recipe["height"], recipe["width"], recipe["iseed"], recipe["kind"]))
    out, seen = {}, {}
    if trace:  # the two volume terms of the (last) forward, for the ratio main() prints
        m.s_lsa.register_forward_hook(lambda mod, inp, res: seen.update(extra=m.gamma * res, f1=inp[1], f2=inp[2]))
    with torch.no_grad():
        if recipe["warm"]:
            from ptlflow.utils.utils import forward_interpolate_batch

            first = m({"images": img})
            out["prev_flow_small"] = LL.np32(first["flow_small"])
            out["flow_init"] = LL.np32(forward_interpolate_batch(first["flow_small"]))
            res = m({"images": img, "prev_preds": {"flow_small": first["flow_small"]}})
        else:
            res = m({"images": img})
    out["flows"] = LL.np32(res["flows"])
    out["flow_small"] = LL.np32(res["flow_small"])
    if trace:
        plain = sys.modules["ptlflow.models.llaflow.corr"].CorrBlock.corr(seen["f1"], seen["f2"])
        out["extra_ratio"] = np.float32(seen["extra"].abs().max() / plain.abs().max())
    return out


def main() -> None:
    if not ref_shim.available():
        raise SystemExit("the reference checkout is not available")
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    mod = load_llaflow()
    for model in ("llaflow", "llaflow_raft"):
        sd = getattr(mod, model)().state_dict()
        with open(os.path.join(GOLDEN_DIR, f"state_shapes_{model}.json"), "w") as f:
            json.dump({k: list(v.shape) for k, v in sd.items()}, f, indent=0)
    import llaflow_oracle as LL

    ops = reference_ops()
    sd, x = LL.op_inputs()
    with torch.no_grad():
        plain, extra = LL.volume(sd, x["fmap1"], x["fmap2"], x["inp"])
    ops["extra_ratio"] = np.float32(extra.abs().max() / plain.abs().max())
    np.savez_compressed(os.path.join(GOLDEN_DIR, "op_llaflow.npz"), recipe=_recipe(seed=LL.OP_SEED), **ops)
    print("op_llaflow", "max|gamma corr2| / max|plain| = %.3f" % ops["extra_ratio"])
    for case in LL.E2E_CASES:
        rec = LL.recipe_of(case)
        out = reference_e2e(rec, trace=True)
        np.savez_compressed(os.path.join(GOLDEN_DIR, case[0] + ".npz"), recipe=_recipe(**rec), **out)
        print(case[0], {k: v.shape for k, v in out.items()}, "max|flow| %.2f" % float(np.abs(out["flows"]).max()),
              "max|gamma corr2| / max|plain| = %.3f" % out["extra_ratio"])


if __name__ == "__main__":
    main()
