"""GPU: LLA-Flow's kernels (both attention tables, the local aggregation, the GEMM operands, the shifted-volume wgmma kernel and the
dense fallback) against float64 with per-element bounds, the operators against the reference fixture, the fp32 fixtures (eager and graph
replay), alternate_corr, the reduction to gma / raft with both gammas at 0, the two volume paths, half precision at 436x1024 against the
fp32 model, and the host errors."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import llaflow_oracle as LL  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(HERE, "golden")
U = {torch.float32: 0.0, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}  # unit roundoff of the storage type
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
HALF = [torch.float16, torch.bfloat16]
F32U = 2.0 ** -24


def _model(name, sd, dtype=torch.float32, **kw):
    from ptlflow_b200.models.llaflow.llaflow import llaflow, llaflow_raft

    m = {"llaflow": llaflow, "llaflow_raft": llaflow_raft}[name](**kw)
    m.load_state_dict(sd)
    return m.eval().to(DEV).to(dtype)


def _pm(x):  # NCHW -> pixel-major
    return x.permute(0, 2, 3, 1).contiguous()


def _rand(shape, dtype, seed, relu=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*shape, generator=g)
    return (x.relu() if relu else x).to(DEV, dtype)


def _taps(x, H, W):
    """pixel-major [B,H,W,C] float64 -> [B,H,W,25,C], tap l at (clamp(y + l // 5 - 2), clamp(x + l % 5 - 2))."""
    ys, xs = torch.arange(H, device=x.device), torch.arange(W, device=x.device)
    return torch.stack([x[:, (ys + l // 5 - 2).clamp(0, H - 1)][:, :, (xs + l % 5 - 2).clamp(0, W - 1)] for l in range(25)], 3)


@pytest.mark.parametrize("dtype", DTYPES)
def test_local_similar_against_float64(dtype):
    from ptlflow_b200 import ops

    B, H, W = 2, 7, 11
    qk = _rand((B, H, W, 512), dtype, 1) * 0.5
    a1, a2 = ops.local_similar(qk)
    x = qk.double()
    for t, got in enumerate((a1, a2)):
        q, k = x[..., 256 * t:256 * t + 128], _taps(x[..., 256 * t + 128:256 * t + 256], H, W)
        logits = torch.einsum("bhwc,bhwlc->bhwl", q, k) / 128 ** 0.5
        ref = torch.softmax(logits, -1).reshape(B * H * W, 25)
        mag = torch.einsum("bhwc,bhwlc->bhwl", q.abs(), k.abs()).reshape(B * H * W, 25).amax(1, keepdim=True) / 128 ** 0.5
        bound = ref * (4 * 128 * F32U * mag + 64 * F32U) + 1e-30  # relative error of the logits' fp32 sums, exp and the division
        assert ((got.double() - ref).abs() <= bound).all(), (got.double() - ref).abs().max().item()


@pytest.mark.parametrize("dtype", DTYPES)
def test_local_aggregate_against_float64(dtype):
    from ptlflow_b200 import ops

    B, H, W = 2, 6, 9
    f2, v = _rand((B, H, W, 256), dtype, 2), _rand((B, H, W, 256), dtype, 3)
    a2 = torch.softmax(_rand((B * H * W, 25), torch.float32, 4), -1)
    gamma = 0.6
    got = ops.local_aggregate(f2, v, a2, gamma).double()
    vt = _taps(v.double(), H, W)
    a = a2.double().view(B, H, W, 25, 1)
    ref = f2.double() + gamma * (a * vt).sum(3)
    bound = U[dtype] * ref.abs() + 32 * F32U * (f2.double().abs() + gamma * (a * vt.abs()).sum(3)) + 1e-30
    assert ((got - ref).abs() <= bound).all()


def _pack_inputs(dtype, B, H, W, seed=5):
    fmap1, f1, fmap2p, f2 = (_rand((B, H, W, 256), dtype, seed + i) for i in range(4))
    a1 = torch.softmax(_rand((B * H * W, 25), torch.float32, seed + 4) * 2, -1)
    return fmap1, f1, a1, fmap2p, f2


def _operands64(fmap1, f1, a1, fmap2p, f2, gamma):
    """float64 A' and B' [B,H,W,6656] of the (rounded) inputs."""
    B, H, W, _ = fmap1.shape
    a = a1.double().view(B, H, W, 25, 1)
    A = torch.cat([fmap1.double()[:, :, :, None] / 16, gamma * a * _taps(f1.double(), H, W) / 16], 3).reshape(B, H, W, 6656)
    Bm = torch.cat([fmap2p.double()[:, :, :, None], _taps(f2.double(), H, W)], 3).reshape(B, H, W, 6656)
    return A, Bm


@pytest.mark.parametrize("dtype", DTYPES)
def test_shift_pack_against_float64(dtype):
    from ptlflow_b200 import ops

    B, H, W, gamma = 2, 5, 7, 0.7
    ins = _pack_inputs(dtype, B, H, W)
    A, Bpad = ops.shift_pack(*ins, gamma, padded=True)
    A2, Bm = ops.shift_pack(*ins, gamma, padded=False)
    rA, rB = _operands64(*ins, gamma)
    assert torch.equal(A, A2)
    # f16: small gamma a1 f1' / 16 entries are subnormal (spacing 2^-24)
    sub = 2.0 ** -25 if dtype == torch.float16 else 0.0
    assert ((A.double() - rA).abs() <= (U[dtype] + 4 * F32U) * rA.abs() + sub + 1e-30).all()
    assert torch.equal(Bm.double(), rB)  # copies
    ys, xs = (torch.arange(H + 4, device=DEV) - 2).clamp(0, H - 1), (torch.arange(W + 4, device=DEV) - 2).clamp(0, W - 1)
    ref_pad = torch.cat([ins[3], ins[4]], 3)[:, ys][:, :, xs]
    assert torch.equal(Bpad, ref_pad)


def _volume64(A, Bm):
    B, H, W, K = A.shape
    return torch.bmm(A.reshape(B, H * W, K), Bm.reshape(B, H * W, K).transpose(1, 2)).reshape(B * H * W, H, W)


def _pool64(v, levels):
    out = [v]
    for _ in range(levels - 1):
        x = out[-1]
        h, w = x.shape[-2] // 2, x.shape[-1] // 2
        x = x[:, : 2 * h, : 2 * w]
        out.append(0.25 * (x[:, 0::2, 0::2] + x[:, 0::2, 1::2] + x[:, 1::2, 0::2] + x[:, 1::2, 1::2]))
    return out


@pytest.mark.parametrize("levels", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("H, W", [(13, 21), (10, 30), (17, 17)])
def test_shift_volume_tiled_against_float64_and_fallback(H, W, dtype, levels):
    """Grids with W not a multiple of 8 or 16 and H not a multiple of 4 or 8, B = 2: the untiled valid cells of every level against
    float64 of the same operands (per-element bound: one rounding plus fp32 accumulation over K = 6656) and against the dense
    fallback (pfb_corr_volume_build_ex on the materialised operands)."""
    from ptlflow_b200 import ops

    B, gamma = 2, 0.7
    ins = _pack_inputs(dtype, B, H, W, seed=H * W)
    A, Bpad = ops.shift_pack(*ins, gamma, padded=True)
    _, Bm = ops.shift_pack(*ins, gamma, padded=False)
    got = ops.shift_volume_tiled(A, Bpad, levels)
    dense = ops.corr_volume_build_ex(A, Bm, levels, scale=1.0, impl=1)
    ref = _pool64(_volume64(A.double(), Bm.double()), levels)
    mag = _pool64(_volume64(A.double().abs(), Bm.double().abs()), levels)
    for l in range(levels):
        h, w = H >> l, W >> l
        t = ops.untile_level(got[l], h, w).double()
        bound = U[dtype] * ref[l].abs() + 2 * 6656 * F32U * mag[l] + 1e-30
        assert ((t - ref[l]).abs() <= bound).all(), (l, (t - ref[l]).abs().max().item())
        assert ((t - dense[l].double()).abs() <= 2 * bound).all(), l


def _engine_ops(m, x, dtype):
    """(a1, a2, fmap2', level 0 of the volume) of the op fixture's inputs through the model's engine."""
    from ptlflow_b200 import ops

    eng = m._get_engine(dtype, torch.device(DEV))
    f1, f2, inp = (_pm(x[k]).to(DEV, dtype) for k in ("fmap1", "fmap2", "inp"))
    B, H, W, _ = f1.shape
    qk = ops.conv2d([inp], eng.ls_qk, torch.empty((B, H, W, 512), dtype=dtype, device=DEV))
    a1, a2 = ops.local_similar(qk)
    f2p = ops.local_aggregate(f2, ops.conv2d([f2], eng.lsa_v, torch.empty_like(f2)), a2, eng.lsa_gamma)
    pyr, layout = eng.lla_volume(f1, f2, inp)
    vol = ops.untile_level(pyr[0], H, W) if layout == 1 else pyr[0]
    return a1, a2, f2p, vol


@pytest.mark.parametrize("dtype", DTYPES)
def test_operators_match_reference_fixture(dtype):
    g = np.load(os.path.join(GOLDEN, "op_llaflow.npz"))
    sd, x = LL.op_inputs()
    m = _model("llaflow", sd, dtype, iters=1)
    a1, a2, f2p, vol = _engine_ops(m, x, dtype)
    B, _, H, W = x["fmap1"].shape
    tol = {torch.float32: 1e-4, torch.float16: 2e-2, torch.bfloat16: 1.5e-1}[dtype]
    ref_vol = torch.from_numpy(g["volume"]).reshape(B * H * W, H, W)
    for got, key, scale in ((a1, "a1", 1.0), (a2, "a2", 1.0), (f2p.permute(0, 3, 1, 2), "fmap2p", 4.0), (vol, "volume", float(ref_vol.abs().max()))):
        ref = torch.from_numpy(g[key]).reshape(got.shape)
        err = (got.float().cpu() - ref).abs().max().item()
        print(f"llaflow {dtype} {key}: max-abs {err:.3g} (scale {scale:.3g})")
        assert err <= tol * scale, key


@pytest.mark.parametrize("name", LL.E2E)
def test_fp32_fixtures_eager_and_replayed(name):
    rec = LL.recipe_of(LL.E2E_CASES[LL.E2E.index(name)])
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    sd, img, kw = LL.e2e_inputs(rec)
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
        assert err < 1e-3, err
        assert (o["flow_small"].cpu() - torch.from_numpy(g["flow_small"])).abs().max().item() < 1e-3


@pytest.mark.parametrize("dtype", DTYPES)
def test_alternate_corr_is_ignored(dtype):
    """alternate_corr=True never takes the on-the-fly lookup (kernel class 3) and gives the flow of False, within the run-to-run
    spread of the forward (its encoders are not bitwise reproducible)."""
    from ptlflow_b200 import _lib

    lib = _lib.load()
    rec = LL.recipe_of(LL.E2E_CASES[LL.E2E.index("e2e_llaflow_default")])
    sd, img, kw = LL.e2e_inputs(rec)
    m = _model("llaflow", sd, dtype, iters=3)
    m.use_cuda_graph = False
    outs = {}
    with torch.no_grad():
        m({"images": img.to(DEV, dtype)})  # the first forward of a shape runs the encoders serially (RAFT._encode)
        for alt in (False, True):
            m.alternate_corr = alt
            n0 = lib.pfb_launch_count(3)
            outs[alt] = m({"images": img.to(DEV, dtype)})["flows_fp32"]
            assert lib.pfb_launch_count(3) == n0
    err = (outs[True] - outs[False]).abs().max().item()
    print(f"llaflow {dtype}: alternate_corr True vs False, max-abs {err:.3g} px")
    assert err < {torch.float32: 1e-4, torch.float16: 1e-2, torch.bfloat16: 5e-2}[dtype]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name, base", [("llaflow", "gma"), ("llaflow_raft", "raft")])
def test_zero_gammas_reduce_to_base_model(name, base, dtype):
    """With gamma = lsa.gamma = 0 the volume is RAFT's: llaflow is gma (one head, content attention), llaflow_raft is raft."""
    import ptlflow_b200 as pb

    sd = LL.synth_state_dict(name, 4, 7)
    sd["gamma"].zero_()
    sd["lsa.gamma"].zero_()
    img = torch.from_numpy(LL.synth.synth_images(1, 128, 160, 8, "smooth")).to(DEV, dtype)
    m = _model(name, sd, dtype, iters=4)
    b = pb.get_model(base)
    b.iters = 4
    bsd = b.state_dict()
    # gma's Attention has a position embedding that content attention never reads; llaflow's has none
    assert {k for k in bsd if k not in sd} <= {k for k in bsd if ".pos_emb." in k}
    b.load_state_dict({**bsd, **{k: v for k, v in sd.items() if k in bsd}}, strict=True)
    b = b.eval().to(DEV).to(dtype)
    with torch.no_grad():
        o1, o2 = m({"images": img})["flows_fp32"], b({"images": img})["flows_fp32"]
    err = (o1 - o2).abs().max().item()
    print(f"{name} with zero gammas vs {base}, {dtype}: max-abs {err:.3g} px")
    assert err < {torch.float32: 1e-4, torch.float16: 1e-2, torch.bfloat16: 5e-2}[dtype]


@pytest.mark.parametrize("dtype", HALF)
def test_tiled_and_dense_volumes_agree(dtype, monkeypatch):
    """Radius 4 in half precision takes the shifted-volume kernel; with the tiled pyramid switched off, A' B'^T on SIMT."""
    from ptlflow_b200 import engine

    rec = LL.recipe_of(LL.E2E_CASES[LL.E2E.index("e2e_llaflow_default")])
    g = torch.from_numpy(np.load(os.path.join(GOLDEN, "e2e_llaflow_default.npz"))["flows"])
    sd, img, kw = LL.e2e_inputs(rec)
    outs = {}
    for tiled in (True, False):
        monkeypatch.setattr(engine, "_TILED", tiled)
        m = _model("llaflow", sd, dtype, **kw)
        m.use_cuda_graph = False
        f = torch.zeros(1, 16, 20, 256, device=DEV, dtype=dtype)
        assert m._get_engine(dtype, torch.device(DEV)).lla_volume(f, f, torch.zeros(1, 16, 20, 128, device=DEV, dtype=dtype))[1] == int(tiled)
        with torch.no_grad():
            outs[tiled] = m({"images": img.to(DEV, dtype)})["flows_fp32"].float().cpu()
    tol = {torch.float16: 0.1, torch.bfloat16: 0.6}[dtype]
    for tiled, o in outs.items():
        e = (o - g).abs().max().item()
        print(f"llaflow {dtype} {'tiled' if tiled else 'dense'} vs the fp32 fixture: max-abs {e:.4f} px")
        assert e < tol
    assert (outs[True] - outs[False]).abs().max().item() < tol


# half precision against the fp32 model at 436 x 1024, 12 iterations (max-abs / mean-abs px)
HALF_GATES = {torch.float16: (8e-2, 2e-2), torch.bfloat16: (5e-1, 1e-1)}


@pytest.mark.parametrize("name", ["llaflow", "llaflow_raft"])
def test_half_precision_at_full_size(name):
    sd = LL.synth_state_dict(name, 4, 5)
    img = torch.from_numpy(LL.synth.synth_images(1, 436, 1024, 6, "smooth")).to(DEV)
    with torch.no_grad():
        ref = _model(name, sd, iters=12)({"images": img})["flows"].float()
        for dtype, bound in HALF_GATES.items():
            out = _model(name, sd, dtype, iters=12)({"images": img.to(dtype)})["flows_fp32"].float()
            e = (out - ref).abs()
            print(f"{name} {dtype} at 436x1024, 12 iterations: max-abs {e.max().item():.4f} mean-abs {e.mean().item():.5f} px "
                  f"(max |flow| {ref.abs().max().item():.1f})")
            assert e.max().item() < bound[0] and e.mean().item() < bound[1]


def test_host_errors_before_any_launch():
    from ptlflow_b200 import _lib

    lib = _lib.load()
    m = _model("llaflow", LL.synth_state_dict("llaflow", 4, 1), iters=2)
    n0 = lib.pfb_launch_count(-1)
    for h, w in ((96, 128), (128, 96)):
        with pytest.raises(ValueError, match="llaflow needs"):
            m({"images": torch.zeros(1, 2, 3, h, w, device=DEV)})
    assert lib.pfb_launch_count(-1) == n0
