"""GPU: CSFlow's strip kernels (means, the two strip GEMMs on SIMT and wgmma, the separable tables with the initial flow, the strip
lookup) against float64 with per-element bounds, the strip operators and the update iteration against the reference fixture, the fp32
fixtures (eager and graph replay), both volume layouts, half precision at 436x1024 against the fp32 model, and the host errors."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import csflow_oracle as CS  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(HERE, "golden")
# unit roundoff of the storage type (one rounding to nearest)
U = {torch.float32: 0.0, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
F32U = 2.0 ** -24


def _model(sd, dtype=torch.float32, **kw):
    import ptlflow_b200 as pb
    from argparse import Namespace

    m = pb.get_model("csflow", args=Namespace(model=Namespace(**kw)) if kw else None)
    m.load_state_dict(sd)
    return m.eval().to(DEV).to(dtype)


def _pm(x):  # NCHW -> pixel-major
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("dtype", DTYPES)
def test_strip_means_against_float64(dtype):
    from ptlflow_b200 import ops

    g = torch.Generator().manual_seed(1)
    B, H, W, C = 2, 17, 23, 256
    gw, gh = (torch.randn(B, H, W, C, generator=g).relu().to(DEV, dtype) for _ in range(2))
    kw, kh = ops.strip_means(gw, gh)
    rw, rh = gw.double().mean(1, keepdim=True), gh.double().mean(2, keepdim=True)
    for got, ref, src, n in ((kw, rw, gw, H), (kh, rh, gh, W)):
        mag = src.double().abs().mean(1 if n == H else 2, keepdim=True)
        bound = U[dtype] * ref.abs() + 2 * n * F32U * mag + 1e-30
        assert ((got.double() - ref).abs() <= bound).all()


@pytest.mark.parametrize("impl", [1, 2])
@pytest.mark.parametrize("dtype", DTYPES)
def test_strip_gemms_against_float64(dtype, impl):
    """sw and sh through pfb_corr_volume_build_ex with scale 1 and a 1 x W / H x 1 target grid, on SIMT (impl 1) and wgmma (impl 2)."""
    from ptlflow_b200 import ops

    if impl == 2 and dtype == torch.float32:
        pytest.skip("wgmma serves f16 / bf16")
    g = torch.Generator().manual_seed(2)
    B, H, W, C = 2, 17, 23, 256
    f1 = torch.randn(B, H, W, C, generator=g).relu().to(DEV, dtype)
    kw, kh = torch.randn(B, 1, W, C, generator=g).relu().to(DEV, dtype), torch.randn(B, H, 1, C, generator=g).relu().to(DEV, dtype)
    for k, n in ((kw, W), (kh, H)):
        out = ops.corr_volume_build_ex(f1, k, 1, scale=1.0, impl=impl)[0]
        assert out.shape == ((B * H * W, 1, W) if n == W else (B * H * W, H, 1))
        ref = torch.einsum("bhwc,bnc->bhwn", f1.double(), k.double().reshape(B, n, C)).reshape(B * H * W, n)
        mag = torch.einsum("bhwc,bnc->bhwn", f1.double().abs(), k.double().abs().reshape(B, n, C)).reshape(B * H * W, n)
        bound = U[dtype] * ref.abs() + 4 * C * F32U * mag + 1e-30
        assert ((out.reshape(B * H * W, n).double() - ref).abs() <= bound).all()


def _strip_inputs(dtype, B=2, H=19, W=23, seed=3):
    g = torch.Generator().manual_seed(seed)
    sw = (torch.rand(B * H * W, W, generator=g) * 4 - 1).to(DEV, dtype)
    sh = (torch.rand(B * H * W, H, generator=g) * 4 - 1).to(DEV, dtype)
    return sw, sh


@pytest.mark.parametrize("dtype", DTYPES)
def test_strip_prepare_against_float64(dtype):
    from ptlflow_b200 import ops

    B, H, W = 2, 19, 23
    sw, sh = _strip_inputs(dtype)
    coords = (CS.O.coords_grid(B, H, W).permute(0, 2, 3, 1) + 0.25).contiguous().to(DEV)
    c0 = coords.clone()
    tw, th = ops.strip_prepare(sw, sh, (H, W), 4, coords)
    for tab, src, n in ((tw, sw, W), (th, sh, H)):
        lvl, off = src.double(), 0
        for l in range(4):
            nl = n >> l
            assert lvl.shape[1] == nl
            got = tab[:, off:off + nl].double()
            assert ((got - lvl).abs() <= 4 * F32U * src.double().abs().amax(1, keepdim=True) + 1e-30).all(), (n, l)
            off += nl
            lvl = 0.5 * (lvl[:, 0:2 * (nl // 2):2] + lvl[:, 1:2 * (nl // 2):2])
        assert off == tab.shape[1]
    init = torch.stack([sh.double().sum(1), sw.double().sum(1)], 1).view(B, H, W, 2)
    mag = torch.stack([sh.double().abs().sum(1), sw.double().abs().sum(1)], 1).view(B, H, W, 2)
    err = (coords.double() - c0.double() - init).abs()
    assert (err <= 2 * max(H, W) * F32U * (mag + c0.double().abs()) + 1e-30).all()
    # without coordinates only the tables are written
    tw2, th2 = ops.strip_prepare(sw, sh, (H, W), 4)
    assert torch.equal(tw2, tw) and torch.equal(th2, th)


def _strip_lookup_ref(sw, sh, coords, r, H, W):
    """float64: the strip channel materialised [Q, H, W], pooled in 2D (raft_oracle.corr_pyramid), sampled bilinearly with zero padding."""
    Q = sw.shape[0]
    S = (sw[:, None, :] + sh[:, :, None]).view(Q, 1, H, W)
    pyr = CS.O.corr_pyramid(S, 4)
    k = 2 * r + 1
    d = torch.arange(-r, r + 1, dtype=torch.float64)
    cx, cy = coords[:, 0].view(Q, 1, 1), coords[:, 1].view(Q, 1, 1)
    outs = []
    for l, v in enumerate(pyr):
        px = (cx / 2**l + d.view(1, k, 1)).expand(Q, k, k).reshape(Q, k * k)
        py = (cy / 2**l + d.view(1, 1, k)).expand(Q, k, k).reshape(Q, k * k)
        outs.append(CS.O._bilinear_zero(v[:, 0], px, py))
    return torch.cat(outs, 1)


@pytest.mark.parametrize("r", [0, 1, 4, 15])
@pytest.mark.parametrize("dtype", DTYPES)
def test_strip_lookup_against_float64(dtype, r):
    """At an odd grid, with fractional, integer, edge and far-out-of-range coordinates, written at an offset that is not 16-byte aligned."""
    from ptlflow_b200 import ops

    B, H, W = 2, 19, 23
    sw, sh = _strip_inputs(dtype, seed=10 + r)
    g = torch.Generator().manual_seed(r)
    coords = torch.rand(B, H, W, 2, generator=g) * torch.tensor([W + 24.0, H + 24.0]) - 12.0
    coords[0, 0, :8, 0] = torch.tensor([0.0, 1.0, W - 1.0, float(W), -1.0, -1e9, 3e9, 12.0])
    coords[0, 1, :8, 1] = torch.tensor([0.0, 1.0, H - 1.0, float(H), -1.0, 5e8, -7e9, 3.0])
    coords = coords.to(DEV)
    tw, th = ops.strip_prepare(sw, sh, (H, W), 4)
    planes = 4 * (2 * r + 1) ** 2
    off = planes + 4  # 8-byte offset in f16 / bf16
    out = torch.full((B, H, W, off + planes + 3), 7.0, dtype=dtype, device=DEV)
    ops.strip_lookup(tw, th, coords, r, 4, out=out, out_offset=off)
    got = out.view(-1, out.shape[-1]).double().cpu()
    ref = _strip_lookup_ref(sw.double().cpu(), sh.double().cpu(), coords.view(-1, 2).double().cpu(), r, H, W)
    mag = (sw.double().abs().amax(1) + sh.double().abs().amax(1)).cpu()[:, None]
    bound = U[dtype] * ref.abs() + 16 * F32U * mag + 1e-30
    assert ((got[:, off:off + planes] - ref).abs() <= bound).all(), ((got[:, off:off + planes] - ref).abs() / bound).max().item()
    assert (got[:, :off] == 7.0).all() and (got[:, off + planes:] == 7.0).all()  # nothing outside its channels
    assert torch.isfinite(got).all()
    assert not got.view(B, H, W, -1)[0, 0, 5:7, off:off + planes].any()  # far out of range (x) reads nothing


def _engine(dtype, impl=0, radius=4):
    sd, x = CS.op_inputs()
    m = _model(sd, dtype, corr_radius=radius)
    m.kernel_impl = impl
    return m, m._get_engine(dtype, torch.device(DEV)), x


@pytest.mark.parametrize("dtype", DTYPES)
def test_strip_operators_match_reference(dtype):
    """The engine's strip maps, the initial flow and the loop's two-channel lookup (RAFT's dense lookup + the strip lookup, permuted to
    the reference's per-level order) against op_csflow.npz."""
    from ptlflow_b200 import ops
    from ptlflow_b200.engine import csflow_convc1_permutation

    g = np.load(os.path.join(GOLDEN, "op_csflow.npz"))
    m, eng, x = _engine(dtype)
    f1, f2 = _pm(x["f1"]).to(DEV, dtype), _pm(x["f2"]).to(DEV, dtype)
    H, W = CS.OP_GRID
    sw, sh = eng.strip_maps(f1, f2)
    ref_sw, ref_sh = torch.from_numpy(g["sw"]), torch.from_numpy(g["sh"])
    tol = {torch.float32: 1e-5, torch.float16: 2e-3, torch.bfloat16: 1e-2}[dtype] * max(ref_sw.abs().max().item(), 1e-3) * 10
    assert (sw.float().cpu().view(ref_sw.shape) - ref_sw).abs().max() < tol
    assert (sh.float().cpu().view(ref_sh.shape) - ref_sh).abs().max() < tol
    coords = _pm(CS.O.coords_grid(1, H, W)).to(DEV)
    tw, th = ops.strip_prepare(sw, sh, (H, W), 4, coords)
    init = coords.permute(0, 3, 1, 2).cpu() - CS.O.coords_grid(1, H, W)
    assert (init - torch.from_numpy(g["corr_init"])).abs().max() < tol * max(H, W)
    if dtype == torch.float32:
        r = CS.OP_LOOKUP_RADIUS
        kk = (2 * r + 1) ** 2
        c = _pm(x["coords"]).to(DEV)
        buf = torch.empty(1, H, W, 8 * kk, device=DEV)
        buf[..., :4 * kk] = ops.corr_lookup(ops.corr_volume_build(f1, f2, 4), c, r, (H, W), nchw=False)
        ops.strip_lookup(tw, th, c, r, 4, out=buf, out_offset=4 * kk)
        ref = torch.from_numpy(g[f"lookup_r{r}"])[:, csflow_convc1_permutation(4, r)]
        assert (buf.permute(0, 3, 1, 2).cpu() - ref).abs().max() < 1e-4


@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES)
def test_update_iteration_matches_reference(dtype, impl):
    """One update iteration with the reference's lookup values, permuted into the buffer's order (convc1 is packed permuted)."""
    from ptlflow_b200.engine import csflow_convc1_permutation

    if dtype == torch.float32 and impl == 0:
        pytest.skip("fp32 runs on SIMT under every impl")
    g = np.load(os.path.join(GOLDEN, "op_csflow.npz"))
    m, eng, x = _engine(dtype, impl)
    hi, wi = CS.OP_ITER_GRID
    net = _pm(x["net"]).to(DEV, dtype)
    coords = _pm(CS.O.coords_grid(1, hi, wi) + x["flow"]).to(DEV)
    corr = _pm(x["corr"][:, csflow_convc1_permutation(4, 4)]).to(DEV, dtype)
    mask = eng.update_iter(net, _pm(x["inp"]).to(DEV, dtype), coords, corr=corr, want_mask=True)
    tol = {torch.float32: 1e-3, torch.float16: 5e-2, torch.bfloat16: 3e-1}[dtype]
    assert (net.permute(0, 3, 1, 2).float().cpu() - torch.from_numpy(g["net"])).abs().max() < tol
    assert (mask.permute(0, 3, 1, 2).float().cpu() - torch.from_numpy(g["mask"])).abs().max() < 4 * tol
    delta = coords.permute(0, 3, 1, 2).cpu() - CS.O.coords_grid(1, hi, wi) - x["flow"]
    assert (delta - torch.from_numpy(g["delta"])).abs().max() < 4 * tol


@pytest.mark.parametrize("name", CS.E2E)
def test_fp32_fixtures_eager_and_replayed(name):
    rec = CS.recipe_of(CS.E2E_CASES[CS.E2E.index(name)])
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    sd, img, kw = CS.e2e_inputs(rec)
    m = _model(sd, **kw)
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
        assert err < 1e-3, err
        assert (o["flow_small"].cpu() - torch.from_numpy(g["flow_small"])).abs().max().item() < 1e-3


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dense_and_tiled_volumes_agree(dtype, monkeypatch):
    """Radius 4 in half precision takes the tiled pyramid; with it switched off the dense one.  Both against the fp32 fixture."""
    from ptlflow_b200 import engine

    rec = CS.recipe_of(CS.E2E_CASES[CS.E2E.index("e2e_csflow_default")])
    g = torch.from_numpy(np.load(os.path.join(GOLDEN, "e2e_csflow_default.npz"))["flows"])
    sd, img, kw = CS.e2e_inputs(rec)
    outs = {}
    for tiled in (True, False):
        monkeypatch.setattr(engine, "_TILED", tiled)
        m = _model(sd, dtype, **kw)
        m.use_cuda_graph = False
        eng = m._get_engine(dtype, torch.device(DEV))
        f = torch.zeros(1, 16, 20, 256, device=DEV, dtype=dtype)
        assert eng.build_volume(f, f)[1] == int(tiled)
        with torch.no_grad():
            outs[tiled] = m({"images": img.to(DEV, dtype)})["flows_fp32"].float().cpu()
    tol = {torch.float16: 0.05, torch.bfloat16: 0.4}[dtype]
    for tiled, o in outs.items():
        e = (o - g).abs()
        print(f"csflow {dtype} {'tiled' if tiled else 'dense'} vs the fp32 fixture: max-abs {e.max().item():.4f} px")
        assert e.max().item() < tol
    assert (outs[True] - outs[False]).abs().max().item() < tol


# the project's half-precision gates against the fp32 model at 436 x 1024, 12 iterations (max-abs / mean-abs px)
HALF_GATES = {torch.float16: (8e-2, 2e-2), torch.bfloat16: (5e-1, 1e-1)}


def test_half_precision_at_full_size():
    sd = CS.synth_state_dict(4, 5)
    img = torch.from_numpy(CS.synth.synth_images(1, 436, 1024, 6, "smooth")).to(DEV)
    with torch.no_grad():
        ref = _model(sd, iters=12)({"images": img})["flows"].float()
        for dtype, bound in HALF_GATES.items():
            out = _model(sd, dtype, iters=12)({"images": img.to(dtype)})["flows_fp32"].float()
            e = (out - ref).abs()
            print(f"csflow {dtype} at 436x1024, 12 iterations: max-abs {e.max().item():.4f} mean-abs {e.mean().item():.5f} px "
                  f"(max |flow| {ref.abs().max().item():.1f})")
            assert e.max().item() < bound[0] and e.mean().item() < bound[1]


def test_host_errors_before_any_launch():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    m = _model(CS.synth_state_dict(4, 1), iters=2)
    n0 = lib.pfb_launch_count(-1)
    for h, w in ((96, 128), (128, 96)):
        with pytest.raises(ValueError, match="csflow needs"):
            m({"images": torch.zeros(1, 2, 3, h, w, device=DEV)})
    assert lib.pfb_launch_count(-1) == n0
