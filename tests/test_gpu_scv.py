"""GPU: SCV's k-NN against float64 with a tie-aware rule and a per-element bound, its determinism, the sparse lookup against the oracle
in every storage type, the update iteration of both models against the reference fixture, the fp32 fixtures (eager and graph replay),
half precision against the fp32 model at 436x1024 and scv4 at 1920x1080, and the host errors."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import scv_oracle as S  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(HERE, "golden")
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
F32U = 2.0 ** -24


def _model(model, sd, dtype=torch.float32, **kw):
    import ptlflow_b200 as pb
    from argparse import Namespace

    m = pb.get_model(model, args=Namespace(model=Namespace(**kw)) if kw else None)
    m.load_state_dict(sd)
    return m.eval().to(DEV).to(dtype)


def _pm(x):  # NCHW -> pixel-major
    return x.permute(0, 2, 3, 1).contiguous()


# (B, N, C, k): N below, at and not a multiple of the 64-target tile, k = N, k in {1, 8, 32}, B = 2
# (C = 64, 128, 192, 256: every C the wgmma path accepts; N = 2000 splits the targets across CTAs)
KNN_CASES = [(1, 40, 256, 32), (1, 64, 256, 32), (2, 200, 256, 8), (1, 33, 256, 33 - 1), (1, 32, 256, 32), (2, 130, 64, 1),
             (1, 517, 128, 32), (1, 300, 192, 1), (1, 2000, 256, 32), (2, 1111, 128, 8)]


@pytest.mark.parametrize("impl", [1, 2])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B, N, C, k", KNN_CASES)
def test_knn_against_float64(B, N, C, k, dtype, impl):
    """Every index distinct and in range; its float64 score at least the true k-th score - tau; no target left out above the true k-th
    score + tau; values within the bound; two runs bit-identical.  tau = C u sum_c |a_c b_c| per element (fp32 accumulation of exact
    products)."""
    from ptlflow_b200 import ops

    if impl == 2 and dtype == torch.float32:
        pytest.skip("wgmma serves f16 / bf16 (fp32 is refused, test_knn_impl_selection)")
    g = torch.Generator().manual_seed(N * 31 + k)
    f1 = torch.randn(B, N, C, generator=g).to(DEV, dtype)
    f2 = torch.randn(B, N, C, generator=g).to(DEV, dtype)
    if N >= 64:  # exact duplicates of one target: ties broken by the lower index
        f2[:, 5] = f2[:, 3]
    scale = C ** -0.5
    val, idx = ops.knn_topk(f1, f2, k, scale, impl=impl)
    val2, idx2 = ops.knn_topk(f1, f2, k, scale, impl=impl)
    assert torch.equal(val, val2) and torch.equal(idx, idx2)
    a, t = f1.double().cpu(), f2.double().cpu()
    s = torch.einsum("bnc,bmc->bnm", a, t).reshape(B * N, N)
    tau = (C * F32U * torch.einsum("bnc,bmc->bnm", a.abs(), t.abs())).reshape(B * N, N)
    idx, val = idx.long().cpu(), val.double().cpu()
    assert ((idx >= 0) & (idx < N)).all()
    assert (idx.sort(dim=1).values.diff(dim=1) > 0).all()  # distinct
    kth = s.sort(dim=1, descending=True).values[:, k - 1 : k]
    got = s.gather(1, idx)
    assert (got >= kth - tau.gather(1, idx)).all()
    chosen = torch.zeros_like(s, dtype=torch.bool).scatter_(1, idx, True)
    assert not ((s > kth + tau) & ~chosen).any()
    assert ((val - got * scale).abs() <= tau.gather(1, idx) * scale + 1e-30).all()
    # descending order, ties to the lower target
    v = val.view(B * N, k)
    assert (v[:, :-1] >= v[:, 1:]).all()


def test_knn_impl_selection():
    """impl 0 takes wgmma where it applies and gives exactly what impl 2 gives; the two kernels select the same targets on separated
    scores; impl 2 refuses what the TMA cannot serve; the split-target merge gives the unsplit result."""
    from ptlflow_b200 import _lib, ops

    g = torch.Generator().manual_seed(11)
    f1, f2 = (torch.randn(1, 700, 128, generator=g).to(DEV, torch.bfloat16) for _ in range(2))
    v0, i0 = ops.knn_topk(f1, f2, 16, impl=0)
    v2, i2 = ops.knn_topk(f1, f2, 16, impl=2)
    v1, i1 = ops.knn_topk(f1, f2, 16, impl=1)
    assert torch.equal(v0, v2) and torch.equal(i0, i2)
    assert (i1 == i2).float().mean() > 0.99 and (v1 - v2).abs().max() < 1e-3
    # the split plan: one sample of 700 queries is 11 query blocks, so the targets are split; 64 samples are not
    lib = _lib.load()
    assert lib.pfb_knn_topk_workspace_bytes(f1.data_ptr(), f2.data_ptr(), 1, 700, 128, 16, 2, 2) > 0
    big = f1.repeat(64, 1, 1)
    assert lib.pfb_knn_topk_workspace_bytes(big.data_ptr(), big.data_ptr(), 64, 700, 128, 16, 2, 2) == 0
    vb, ib = ops.knn_topk(big, f2.repeat(64, 1, 1), 16, impl=2)
    assert torch.equal(vb[:700], v2) and torch.equal(ib[:700], i2)
    for bad in (f1.float(), f1[..., :96].contiguous()):
        with pytest.raises(RuntimeError):
            ops.knn_topk(bad, bad, 16, impl=2)


def test_knn_matches_reference_fixture():
    from ptlflow_b200 import ops

    g = np.load(os.path.join(GOLDEN, "op_scv.npz"))
    _, x = S.op_inputs()
    p = S.OP_KNN
    val, idx = ops.knn_topk(_pm(x["f1"]).to(DEV), _pm(x["f2"]).to(DEV), p["k"], p["C"] ** -0.5)
    assert np.array_equal(idx.cpu().numpy().reshape(g["knn_idx"].shape), g["knn_idx"])
    assert np.abs(val.cpu().numpy().reshape(g["knn_val"].shape) - g["knn_val"]).max() < 1e-5


@pytest.mark.parametrize("dtype", DTYPES)
def test_sparse_lookup_against_oracle(dtype):
    """Displacements inside, on and beyond the +-4 edge of every level (op_scv.npz): a table of query + displacement looked up at the
    start grid, against the reference's splat; then sparse_prepare's table of integer targets under a warm start."""
    from ptlflow_b200 import ops

    g = np.load(os.path.join(GOLDEN, "op_scv.npz"))
    _, x = S.op_inputs()
    disp, val = x["disp"], x["val"]  # [1, n, k, 2] (y, x), [1, n, k]
    n, k = disp.shape[1], disp.shape[2]
    H, W = 8, n // 8
    # targets are not needed: a table entry is (ty + wy, tx + wx); build it directly as query + displacement, then check the kernel's
    # own table on integer targets below
    q = torch.arange(n)
    grid = torch.stack([(q % W).float(), (q // W).float()], -1).view(1, H, W, 2)
    table = torch.stack([disp[0, :, :, 0] + grid.view(n, 1, 2)[..., 1], disp[0, :, :, 1] + grid.view(n, 1, 2)[..., 0], val[0]], -1)
    coords = grid.clone().to(DEV)
    stride = 408 if dtype != torch.float32 else 405
    out = ops.sparse_lookup(table.contiguous().to(DEV), coords, dtype, stride)
    ref = torch.from_numpy(g["lookup"])[0]
    tol = {torch.float32: 1e-5, torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}[dtype] * (ref.abs() + 1) * 2
    got = out.view(n, stride).float().cpu()
    assert (got[:, :405] - ref).abs().le(tol).all()
    assert not got[:, 405:].any()
    assert torch.equal(out, ops.sparse_lookup(table.contiguous().to(DEV), coords, dtype, stride))
    # sparse_prepare: integer targets, a warm start of w moves every entry by w
    idx = torch.randint(0, n, (n, k), generator=torch.Generator().manual_seed(7), dtype=torch.int32)
    w = torch.randn(1, H, W, 2, generator=torch.Generator().manual_seed(8))
    tab = ops.sparse_prepare(val[0].contiguous().to(DEV), idx.to(DEV), (grid + w).contiguous().to(DEV)).cpu()
    exp = torch.stack([(idx // W).float() + w.view(n, 1, 2)[..., 1], (idx % W).float() + w.view(n, 1, 2)[..., 0], val[0]], -1)
    assert (tab - exp).abs().max() < 1e-5


def _engine(model, dtype, impl=0):
    sds, x = S.op_inputs()
    m = _model(model, sds[model], dtype)
    m.kernel_impl = impl
    return m, m._get_engine(dtype, torch.device(DEV)), x


@pytest.mark.parametrize("model", S.MODELS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_update_iteration_matches_reference(model, dtype):
    """With the reference's lookup values handed in ([P, 405] rows are not 16-byte aligned in f16 / bf16, so the SIMT convolutions
    read them; the loop's own 408-wide buffer feeds the tensor-core path in the end-to-end tests)."""
    g = np.load(os.path.join(GOLDEN, "op_scv.npz"))
    m, eng, x = _engine(model, dtype, impl=1)
    hi, wi = S.OP_ITER_GRID
    net = _pm(x["net"]).to(DEV, dtype)
    coords = _pm(S.O.coords_grid(1, hi, wi) + x["flow"]).to(DEV)
    corr = _pm(x["corr"]).to(DEV, dtype)
    mask = eng.update_iter(net, _pm(x["inp"]).to(DEV, dtype), coords, corr=corr, want_mask=True)
    tol = {torch.float32: 1e-3, torch.float16: 5e-2, torch.bfloat16: 3e-1}[dtype]
    assert (net.permute(0, 3, 1, 2).float().cpu() - torch.from_numpy(g[f"{model}_net"])).abs().max() < tol
    assert (mask.permute(0, 3, 1, 2).float().cpu() - torch.from_numpy(g[f"{model}_mask"])).abs().max() < 4 * tol
    delta = coords.permute(0, 3, 1, 2).cpu() - S.O.coords_grid(1, hi, wi) - x["flow"]
    assert (delta - torch.from_numpy(g[f"{model}_delta"])).abs().max() < 4 * tol


@pytest.mark.parametrize("name", S.E2E)
def test_fp32_fixtures_eager_and_replayed(name):
    rec = S.recipe_of(S.E2E_CASES[S.E2E.index(name)])
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    sd, img, kw = S.e2e_inputs(rec)
    m = _model(rec["model"], sd, **kw)
    inputs = {"images": img.to(DEV)}
    if rec["warm"]:
        inputs["prev_preds"] = {"flow_small": torch.from_numpy(g["prev_flow_small"]).to(DEV)}
    outs = []
    with torch.no_grad():
        for _ in range(3):  # eager, eager + capture, replay
            outs.append(m(inputs))
    assert m.graph_replays >= 1
    for o in outs:
        err = (o["flows"].cpu() - torch.from_numpy(g["flows"])).abs().max().item()
        print(f"{name}: max-abs {err:.2e} px against the reference")
        assert err < 1e-4, err
        assert (o["flow_small"].cpu() - torch.from_numpy(g["flow_small"])).abs().max().item() < 1e-4


# half precision against the fp32 model on the same card (max-abs / mean-abs px), about 3x the errors measured on an H100 80GB HBM3 at
# 700 W with 12 iterations at 436x1024: f16 0.26 / 0.049 (scv8) and 0.18 / 0.020 (scv4), bf16 1.00 / 0.131 (scv8) and 0.40 / 0.058
# (scv4); scv4 in bf16 at 1080x1920: 0.67 / 0.043
HALF_GATES = {torch.float16: (0.8, 0.15), torch.bfloat16: (3.0, 0.4)}


def _half_vs_fp32(model, h, w, iters, dtypes):
    sd = S.synth_state_dict(model, 5)
    img = torch.from_numpy(S.synth.synth_images(1, h, w, 6, "smooth")).to(DEV)
    with torch.no_grad():
        ref = _model(model, sd, iters=iters)({"images": img})["flows"].float()
        for dtype in dtypes:
            torch.cuda.reset_peak_memory_stats()
            out = _model(model, sd, dtype, iters=iters)({"images": img.to(dtype)})["flows_fp32"].float()
            e = (out - ref).abs()
            print(f"{model} {dtype} at {h}x{w}, {iters} iterations: max-abs {e.max().item():.4f} mean-abs {e.mean().item():.5f} px "
                  f"(max |flow| {ref.abs().max().item():.1f}), peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")
            bound = HALF_GATES[dtype]
            assert e.max().item() < bound[0] and e.mean().item() < bound[1]


@pytest.mark.parametrize("model", S.MODELS)
def test_half_precision_at_full_size(model):
    _half_vs_fp32(model, 436, 1024, 12, (torch.float16, torch.bfloat16))


def test_scv4_bf16_at_1080p():
    """N = 480 x 272 = 130 560 queries: the dense f16 volume would take 34 GB; the k-NN keeps 32 matches of each."""
    _half_vs_fp32("scv4", 1080, 1920, 12, (torch.bfloat16,))


def test_num_k_change_after_capture():
    """Changing num_k after a forward rebuilds the engine and captures a new graph: the result equals a model built with that num_k."""
    rec = S.recipe_of(S.E2E_CASES[S.E2E.index("e2e_scv8_k8")])
    g = np.load(os.path.join(GOLDEN, "e2e_scv8_k8.npz"))
    sd, img, kw = S.e2e_inputs(rec)
    m = _model("scv8", sd, iters=kw["iters"])  # num_k 32
    with torch.no_grad():
        for _ in range(3):
            m({"images": img.to(DEV)})
        m.num_k = 8
        for _ in range(3):
            out = m({"images": img.to(DEV)})
    assert m._engine.num_k == 8
    assert (out["flows"].cpu() - torch.from_numpy(g["flows"])).abs().max().item() < 1e-4


def test_host_errors_before_any_launch():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    m = _model("scv8", S.synth_state_dict("scv8", 1), iters=2)
    n0 = lib.pfb_launch_count(-1)
    with pytest.raises(ValueError, match="num_k=32"):
        m({"images": torch.zeros(1, 2, 3, 32, 48, device=DEV)})  # a 4 x 6 grid
    assert lib.pfb_launch_count(-1) == n0
