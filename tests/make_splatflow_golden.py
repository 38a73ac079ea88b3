"""Write the SplatFlow fixtures under tests/golden/ by running the REAL reference (where its checkout exists).

TEST INFRASTRUCTURE, the counterpart of oracle/make_golden.py for SplatFlow.  Usage, from the repository root:

    python tests/make_splatflow_golden.py

Writes op_splatflow.npz (the splat on crafted flows, and one gru_sp update of the reference's own update.py modules), the
e2e_splatflow_* cases of splatflow_oracle.E2E_CASES and state_shapes_splatflow.json.  Inputs and weights are rebuilt from the
recipes by splatflow_oracle / oracle.synth, so the fixtures hold outputs only.

The reference's splat is a cupy kernel (softsplat.py), and its SplatFlow refuses to construct without cupy.  Here
``splatflow.forward_warping`` is replaced by softsplat_stand_in, a CPU restatement of that kernel (softsplat.py:10-60, 435-468) line
for line: fp32 weights and products, fp64 index_add_, .float() before normalising.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import splatflow_oracle as SO  # noqa: E402
from oracle import fixtures as F  # noqa: E402
from oracle import ref_shim  # noqa: E402


def softsplat_stand_in(tenInput, tenFlow, tenMetric=None, strType="average"):
    """FunctionSoftsplat(tenInput, tenFlow, None, "average") of softsplat.py on the CPU."""
    assert tenMetric is None and strType == "average"
    tenInput = torch.cat([tenInput, tenInput.new_ones(tenInput.shape[0], 1, tenInput.shape[2], tenInput.shape[3])], 1)
    n, c, h, w = tenInput.shape
    output = torch.zeros((n, c, h * w), dtype=torch.float64)
    gy, gx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    fltOutputX = gx.float()[None] + tenFlow[:, 0].float()
    fltOutputY = gy.float()[None] + tenFlow[:, 1].float()
    intNorthwestX, intNorthwestY = torch.floor(fltOutputX).long(), torch.floor(fltOutputY).long()
    intNortheastX, intNortheastY = intNorthwestX + 1, intNorthwestY
    intSouthwestX, intSouthwestY = intNorthwestX, intNorthwestY + 1
    intSoutheastX, intSoutheastY = intNorthwestX + 1, intNorthwestY + 1
    fltNorthwest = (intSoutheastX.float() - fltOutputX) * (intSoutheastY.float() - fltOutputY)
    fltNortheast = (fltOutputX - intSouthwestX.float()) * (intSouthwestY.float() - fltOutputY)
    fltSouthwest = (intNortheastX.float() - fltOutputX) * (fltOutputY - intNortheastY.float())
    fltSoutheast = (fltOutputX - intNorthwestX.float()) * (fltOutputY - intNorthwestY.float())
    value = tenInput.float()
    for cx, cy, wt in ((intNorthwestX, intNorthwestY, fltNorthwest), (intNortheastX, intNortheastY, fltNortheast),
                       (intSouthwestX, intSouthwestY, fltSouthwest), (intSoutheastX, intSoutheastY, fltSoutheast)):
        inside = (cx >= 0) & (cx < w) & (cy >= 0) & (cy < h)
        for b in range(n):
            m = inside[b].reshape(-1)
            prod = (value[b].reshape(c, -1) * wt[b].reshape(1, -1))[:, m]  # value * weight, rounded to fp32
            output[b].index_add_(1, (cy[b] * w + cx[b]).reshape(-1)[m], prod.double())
    tenOutput = output.reshape(n, c, h, w).float()
    tenNormalize = tenOutput[:, -1:, :, :]
    tenNormalize[tenNormalize == 0.0] = 1.0
    return tenOutput[:, :-1, :, :] / tenNormalize


def load_splatflow():
    """-> the reference module ptlflow.models.splatflow.splatflow, with the CPU stand-in as its forward_warping."""
    ref_shim.install()
    lm = sys.modules["lightning.pytorch"].LightningModule
    if "dtype" not in lm.__dict__:
        lm.dtype = property(lambda self: next(self.parameters()).dtype)
        lm.device = property(lambda self: next(self.parameters()).device)
    mod = F.load_package("splatflow", "splatflow").splatflow
    mod.forward_warping = softsplat_stand_in
    return mod


def reference_model(kwargs):
    return F.reference_model(load_splatflow().splatflow(**kwargs), SO.synth_state_dict)


def reference_e2e(recipe):
    """The arrays of an e2e_splatflow_* fixture (with the ignored prev_preds flow_small of a ``prev`` case)."""
    model = F.reference_model(load_splatflow().splatflow(**recipe["kwargs"]), lambda shapes: SO.synth_state_dict(shapes, recipe["wseed"]))
    inputs = {"images": SO.images(recipe)}
    out = {}
    if recipe["prev"]:
        out["prev_flow_small"] = F.np32(SO.prev_flow_small(recipe))
        inputs["prev_preds"] = {"flow_small": SO.prev_flow_small(recipe)}
    with torch.no_grad():
        res = model(inputs)
    out["flows"] = F.np32(res["flows"])
    out["flow_small"] = F.np32(res["flow_small"])
    return out


def reference_ops() -> dict:
    """op_splatflow.npz: the splat of op_splat_inputs and one gru_sp update of the reference's Update module."""
    load_splatflow()
    import ptlflow.models.splatflow.update as up

    x, flow = SO.op_splat_inputs()
    arrays = {"splat": F.np32(softsplat_stand_in(x, flow))}
    sd, net, inp, corr, flow, attn, mf_t = SO.op_iter_inputs()
    blk = up.Update(hidden_dim=128).eval()
    blk.load_state_dict({k[len("update."):]: v for k, v in sd.items() if k.startswith("update.")})
    with torch.no_grad():
        n, m, d, mf = blk(net, inp, corr, flow, attn, mf_t)
    arrays.update(iter_net=F.np32(n), iter_mask=F.np32(m), iter_delta=F.np32(d), iter_mf=F.np32(mf))
    return arrays


def main() -> None:
    F.start()
    F.write_fixture("op_splatflow", dict(seed=SO.OP_SEED), reference_ops())
    for case in SO.E2E_CASES:
        rec = SO.recipe_of(case)
        out = reference_e2e(rec)
        F.write_fixture(case[0], rec, out)
        print(case[0], {k: v.shape for k, v in out.items()}, "max|flow| %.2f" % float(np.abs(out["flows"]).max()))
    F.write_state_shapes("splatflow", load_splatflow().splatflow())


if __name__ == "__main__":
    main()
