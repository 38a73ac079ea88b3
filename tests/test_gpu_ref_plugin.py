"""This library's plugin entry point against the REFERENCE'S OWN native kernel, alt_cuda_corr
(ptlflow/utils/external/alt_cuda_corr of the reference): ``alt_cuda_corr.forward(fmap1, fmap2, coords, radius)`` -- same
tensors in, same tensor out (correlation.cpp:23-33).  The reference kernel's outputs for these inputs are stored in
tests/golden/ref_plugin_alt_corr.npz as a fixed, seeded sample of elements (``python -m oracle.make_golden ref_plugin``)."""
import numpy as np
import pytest

from helpers import load_golden_arrays
from oracle import make_golden as G

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("b,c,h1,w1,h2,w2,r", G.REF_PLUGIN_CASES)
def test_forward_matches_the_reference_kernel(b, c, h1, w1, h2, w2, r):
    from ptlflow_b200 import alt_cuda_corr

    case = G.REF_PLUGIN_CASES.index((b, c, h1, w1, h2, w2, r))
    g = load_golden_arrays("ref_plugin_alt_corr")
    f1, f2, coords = (t.to(DEV) for t in G.ref_plugin_inputs(b, c, h1, w1, h2, w2))
    (ours,) = alt_cuda_corr.forward(f1, f2, coords, r)
    assert tuple(ours.shape) == tuple(g[f"shape{case}"]) and ours.dtype.is_floating_point and ours.element_size() == 4
    flat = ours.cpu().numpy().reshape(-1)
    idx = g[f"idx{case}"]
    assert np.array_equal(idx, G.ref_plugin_sample(flat.size))
    ref = g[f"val{case}"]
    scale = max(1.0, float(np.abs(ref).max()))
    assert float(np.abs(flat[idx] - ref).max()) < 2e-5 * scale, float(np.abs(flat[idx] - ref).max())
