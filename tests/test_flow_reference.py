"""CPU: the bounds of flow_reference.py and of conv_reference's FLOW epilogue admit correct fp32 implementations of the flow
kernels (the models' references and fp32 re-implementations of each kernel's operation order) and reject plausible kernel
bugs on seeded inputs; pfb_conv2d refuses a FLOW output window that cannot hold both flow components."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import ccmr_oracle as CC  # noqa: E402
import conv_reference as R  # noqa: E402
import flow_reference as FR  # noqa: E402
import ms_raft_oracle as MS  # noqa: E402
import scv_oracle as SCV  # noqa: E402
from oracle import raft_oracle as O  # noqa: E402

HALF = [torch.float16, torch.bfloat16]
MASK_DTYPES = [torch.float16, torch.bfloat16, torch.float32]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _coords(B, H, W, seed, amp=60.0):
    """fp32 coordinates [B,H,W,2]: the grid plus a flow of up to ``amp`` px."""
    g = _gen(seed)
    return (FR.grid_xy(B, H, W) + (torch.rand(B, H, W, 2, generator=g, dtype=torch.float64) * 2 - 1) * amp).float()


def _mask(B, H, W, F_, dtype, seed, scale=3.0):
    return (torch.randn(B, H, W, 9 * F_ * F_, generator=_gen(seed)) * scale).to(dtype)


def _fma_chain(terms):
    """fp32 fmaf accumulation of the (value, weight) pairs in order, products exact, each step rounded once."""
    acc = torch.zeros_like(terms[0][0], dtype=torch.float32)
    for a, b in terms:
        acc = (a.double() * b.double() + acc.double()).float()
    return acc


# ------------------------------------------------------------------------------------------------------------------------------
# convex upsample
# ------------------------------------------------------------------------------------------------------------------------------
def convex_fp32(coords, mask, F_, mode=0, swap_sub=False, sub_major=False, drop_oob_denominator=False, no_fine_grid=False):
    """The convex kernels' operation order in fp32 -> [B,2,F H,F W] float32; the keyword arguments are the bugs."""
    B, H, W, _ = coords.shape
    FF = F_ * F_
    m = mask.float().view(B, H, W, 9 * FF)
    g = FR.grid_xy(B, H, W).float() if mode != 1 else torch.zeros_like(coords)
    a = F_ * (coords - g)
    ap = F.pad(a.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    inb = F.pad(torch.ones(B, 1, H, W), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    out = torch.empty(B, H, W, F_, F_, 2)
    for sy in range(F_):
        for sx in range(F_):
            ssy, ssx = (sx, sy) if swap_sub else (sy, sx)
            sub = ssy * F_ + ssx
            v = [m[..., sub * 9 + t] if sub_major else m[..., t * FF + sub] for t in range(9)]
            mx = torch.stack(v, -1).amax(-1)
            s = torch.zeros(B, H, W)
            ax = torch.zeros(B, H, W, 2)
            for t in range(9):
                dy, dx = t // 3, t % 3
                e = torch.exp(v[t] - mx)
                ok = inb[:, dy:dy + H, dx:dx + W, 0]
                s = s + (e * ok if drop_oob_denominator else e)
                ax = (e[..., None].double() * ap[:, dy:dy + H, dx:dx + W].double() + ax.double()).float()
            out[:, :, :, sy, sx] = ax * (1.0 / s)[..., None]
    out = FR.to_nchw(out, F_)
    if mode == 2 and not no_fine_grid:
        out = out + FR.grid_xy(B, F_ * H, F_ * W).permute(0, 3, 1, 2).float()
    return out


def _oracle_convex(coords, mask, F_, mode):
    """The models' references: raft_oracle (8x), scv_oracle (4x), ms_raft_oracle (2x; mode 1 of the absolute coordinates, the
    handover as in ccmr.py), all fp32."""
    B, H, W, _ = coords.shape
    m = mask.float().permute(0, 3, 1, 2)
    grid = O.coords_grid(B, H, W)
    flow = coords.permute(0, 3, 1, 2) - grid
    if F_ == 8:
        return O.convex_upsample(flow, m)
    if F_ == 4:
        return SCV.convex_upsample4(flow, m)
    if mode == 0:
        return MS.convex_up2(flow, m)
    if mode == 1:
        return MS.convex_up2(coords.permute(0, 3, 1, 2), m)
    return O.coords_grid(B, 2 * H, 2 * W) + MS.convex_up2(flow, m)


CONVEX = [(8, 0), (4, 0), (2, 0), (2, 1), (2, 2)]


@pytest.mark.parametrize("F_,mode", CONVEX, ids=[f"x{f}-mode{m}" for f, m in CONVEX])
@pytest.mark.parametrize("dtype", MASK_DTYPES, ids=["f16", "bf16", "f32"])
def test_convex_bound_admits_fp32_implementations(F_, mode, dtype):
    coords = _coords(2, 5, 7, 1 + F_ + mode, amp=300.0)
    mask = _mask(2, 5, 7, F_, dtype, 2 + F_ + mode)
    ref, bound = FR.convex(coords, mask, F_, mode)
    FR.assert_within(convex_fp32(coords, mask, F_, mode), ref, bound, "fp32 kernel order")
    FR.assert_within(_oracle_convex(coords, mask, F_, mode), ref, bound, "oracle")


def test_convex_bound_admits_wide_and_flat_masks():
    """Logits far apart (x_t down to -200: the |x_t| terms) and all equal (the full 9-term sums)."""
    coords = _coords(1, 4, 6, 5, amp=400.0)
    for mask in (_mask(1, 4, 6, 8, torch.float32, 6, scale=60.0), torch.zeros(1, 4, 6, 576)):
        ref, bound = FR.convex(coords, mask, 8)
        FR.assert_within(convex_fp32(coords, mask, 8), ref, bound, "fp32 kernel order")
        FR.assert_within(_oracle_convex(coords, mask, 8, 0), ref, bound, "oracle")


CONVEX_BUGS = ["swap_sub", "sub_major", "drop_oob_denominator"]


@pytest.mark.parametrize("bug", CONVEX_BUGS)
@pytest.mark.parametrize("F_,mode", CONVEX, ids=[f"x{f}-mode{m}" for f, m in CONVEX])
def test_convex_bugs_rejected(bug, F_, mode):
    coords = _coords(2, 5, 7, 11, amp=50.0)
    mask = _mask(2, 5, 7, F_, torch.float16, 12)
    ref, bound = FR.convex(coords, mask, F_, mode)
    assert FR.max_ratio(convex_fp32(coords, mask, F_, mode, **{bug: True}), ref, bound) > 1.0


def test_convex_missing_fine_grid_rejected():
    coords = _coords(1, 4, 5, 13)
    mask = _mask(1, 4, 5, 2, torch.float16, 14)
    ref, bound = FR.convex(coords, mask, 2, 2)
    assert FR.max_ratio(convex_fp32(coords, mask, 2, 2, no_fine_grid=True), ref, bound) > 1.0


@pytest.mark.parametrize("F_", [8, 4, 2])
def test_convex_window_off_by_one_rejected(F_):
    coords = _coords(1, 4, 6, 15)
    mask = _mask(1, 4, 6, F_, torch.float32, 16)
    ref, bound = FR.convex(coords, mask, F_)
    full = convex_fp32(coords, mask, F_)
    oh, ow = F_ * 4 - 2, F_ * 6 - 2
    for (pt, pl), (qt, ql) in (((1, 1), (2, 1)), ((1, 1), (1, 0))):
        win = lambda t, a, b: t[:, :, a:a + oh, b:b + ow]  # noqa: E731
        FR.assert_within(win(full, pt, pl), win(ref, pt, pl), win(bound, pt, pl), "window")
        assert FR.max_ratio(win(full, qt, ql), win(ref, pt, pl), win(bound, pt, pl)) > 1.0


@pytest.mark.parametrize("F_,mode", CONVEX, ids=[f"x{f}-mode{m}" for f, m in CONVEX])
def test_onehot_expected_is_the_gather(F_, mode):
    """A one-hot mask (one logit 0, eight at -120) makes the fp32 kernel order a gather: onehot_expected bit for bit."""
    B, H, W = 2, 3, 4
    coords = _coords(B, H, W, 17, amp=300.0)
    tap = (torch.arange(F_ * F_).view(1, 1, 1, F_, F_) + torch.arange(H * W).view(1, H, W, 1, 1) + 4) % 9
    tap = tap.expand(B, H, W, F_, F_)
    mask = torch.full((B, H, W, 9, F_ * F_), -120.0)
    mask.scatter_(3, tap.reshape(B, H, W, 1, F_ * F_), 0.0)
    mask = mask.view(B, H, W, 9 * F_ * F_).half()
    exp = FR.onehot_expected(coords, tap, F_, mode)
    got = convex_fp32(coords, mask, F_, mode)
    assert torch.equal(R.bits(got), R.bits(exp))
    ref, bound = FR.convex(coords, mask, F_, mode)
    FR.assert_within(exp, ref, bound, "one-hot")


# ------------------------------------------------------------------------------------------------------------------------------
# bilinear resamplers
# ------------------------------------------------------------------------------------------------------------------------------
def _flow(B, H, W, seed, amp=60.0):
    return (torch.rand(B, 2, H, W, generator=_gen(seed), dtype=torch.float64) * 2 - 1).mul(amp).float()


@pytest.mark.parametrize("H,W,out", [(7, 11, (56, 88)), (1, 9, (8, 72)), (9, 1, (72, 8)), (1, 1, (8, 8)), (3, 50, (24, 400))])
def test_source_index_matches_interpolate(H, W, out):
    """The fp32 index arithmetic reproduces F.interpolate: interpolating the column (row) index gives i0 + lam up to the blend's
    rounding, and a blend of random values stays inside the bound."""
    oh, ow = out
    i0, i1, lx = FR.aten_source_index(W, ow, np.arange(ow))
    ramp = torch.arange(W, dtype=torch.float32).view(1, 1, 1, W).expand(1, 1, H, W)
    got = F.interpolate(ramp, size=out, mode="bilinear", align_corners=True)[0, 0, 0].double().numpy()
    want = i0 + (i1 - i0) * lx.astype(np.float64)
    np.testing.assert_allclose(got, want, rtol=0, atol=4 * FR.U24 * max(W, 1))
    f = _flow(2, H, W, H * 100 + W)
    ref, bound = FR.bilinear(f, out)
    FR.assert_within(F.interpolate(f, size=out, mode="bilinear", align_corners=True), ref, bound, "interpolate")


def test_upflow_references_admit_oracles():
    coords = _coords(2, 6, 40, 21, amp=300.0)
    ref, bound = FR.upflow(coords, 8)
    flow = coords.permute(0, 3, 1, 2) - O.coords_grid(2, 6, 40)
    FR.assert_within(O.upflow8(flow), ref, bound, "raft upflow8")
    f = _flow(2, 6, 40, 22, amp=300.0)
    FR.assert_within(CC.upflow2(f), *FR.upflow2(f), "ccmr upflow2")
    f = _flow(2, 55, 128, 23, amp=300.0)
    FR.assert_within(MS.downflow(f), *FR.downflow(f, (3, 8)), "ms_raft downflow")
    for out_hw in ((1, 1), (4, 5), (20, 33)):
        want = F.interpolate(f, size=out_hw, mode="bilinear", align_corners=True)
        su, sv = FR.downflow_scales(55, 128, *out_hw)
        want = torch.cat([want[:, :1] * su, want[:, 1:] * sv], 1)
        FR.assert_within(want, *FR.downflow(f, out_hw), f"downflow {out_hw}")


def _blend_with(f, full_hw, idx):
    """mult-free blend of f with the index function idx(n_in, n_out, o) -> (i0, i1, lam), float64."""
    H, W = f.shape[-2:]
    y0, y1, ly = idx(H, full_hw[0], np.arange(full_hw[0]))
    x0, x1, lx = idx(W, full_hw[1], np.arange(full_hw[1]))
    ly = torch.as_tensor(np.asarray(ly, dtype=np.float64))[:, None]
    lx = torch.as_tensor(np.asarray(lx, dtype=np.float64))[None, :]
    f = f.double()
    r0, r1 = f[:, :, y0], f[:, :, y1]
    return (1 - ly) * ((1 - lx) * r0[..., x0] + lx * r0[..., x1]) + ly * ((1 - lx) * r1[..., x0] + lx * r1[..., x1])


def _idx_f64_scale(n_in, n_out, o):
    src = (n_in - 1) / (n_out - 1) * np.asarray(o, dtype=np.float64) if n_out > 1 else np.zeros(len(o))
    i0 = np.floor(src).astype(np.int64)
    return i0, i0 + (i0 < n_in - 1), src - i0


def _idx_src_rounded_late(n_in, n_out, o):
    """scale * o with the scale and the product in float64 and one rounding to fp32 at the end."""
    src = ((n_in - 1) / (n_out - 1) * np.asarray(o, dtype=np.float64)).astype(np.float32) if n_out > 1 else np.zeros(len(o), np.float32)
    i0 = np.floor(src).astype(np.int64)
    return i0, i0 + (i0 < n_in - 1), (src - i0.astype(np.float32)).astype(np.float64)


def test_upflow8_bound_admits_fp32_kernel_order():
    coords = _coords(2, 6, 100, 31, amp=300.0)
    B, H, W, _ = coords.shape
    ref, bound = FR.upflow(coords, 8)
    f = (coords.permute(0, 3, 1, 2) - O.coords_grid(B, H, W))
    y0, y1, ly = FR.aten_source_index(H, 8 * H, np.arange(8 * H))
    x0, x1, lx = FR.aten_source_index(W, 8 * W, np.arange(8 * W))
    ly, lx = torch.from_numpy(ly)[:, None], torch.from_numpy(lx)[None, :]
    r0, r1 = f[:, :, y0], f[:, :, y1]
    v = (1 - ly) * ((1 - lx) * r0[..., x0] + lx * r0[..., x1]) + ly * ((1 - lx) * r1[..., x0] + lx * r1[..., x1])
    assert v.dtype == torch.float32
    FR.assert_within(8 * v, ref, bound, "fp32 upflow8")


@pytest.mark.parametrize("bug", ["align_corners_false", "f64_scale", "src_rounded_late"])
def test_upflow8_index_bugs_rejected(bug):
    coords = _coords(1, 6, 100, 32, amp=300.0)
    B, H, W, _ = coords.shape
    ref, bound = FR.upflow(coords, 8)
    flow = FR.flow_of(coords)
    if bug == "align_corners_false":
        got = 8 * F.interpolate(flow.float(), size=(8 * H, 8 * W), mode="bilinear", align_corners=False)
    else:
        got = 8 * _blend_with(flow, (8 * H, 8 * W), _idx_f64_scale if bug == "f64_scale" else _idx_src_rounded_late)
    assert FR.max_ratio(got, ref, bound) > 1.0


# ------------------------------------------------------------------------------------------------------------------------------
# flow head
# ------------------------------------------------------------------------------------------------------------------------------
def _head_operands(B, H, W, cin, dtype, seed, amp=400.0):
    g = _gen(seed)
    x = torch.randn(B, H, W, cin, generator=g).to(dtype)
    w = (torch.randn(2, cin, 3, 3, generator=g) * (9 * cin) ** -0.5).to(dtype)
    bias = torch.randn(2, generator=g) * 0.1
    coords = _coords(B, H, W, seed + 1, amp)
    return x, w, bias, coords


def _head_reference(x, w, bias, coords):
    acc, S, n = R.conv_terms([x.double()], w.double(), bias.double())
    return R.epilogue(R.FLOW, acc, S, n, torch.float32, coords=coords.double())


def _neighbour(t, dy, dx):
    """t [B,H,W,C] shifted so that pixel (y, x) reads (y + dy, x + dx), zero outside."""
    H, W = t.shape[1:3]
    tp = F.pad(t.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    return tp[:, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W]


def head_warp_fp32(x, w, bias, coords, drop_chunk=None, bias_twice=False):
    """conv_cout2_flow_kernel's order: lane l takes the 8-channel chunks l, l + 32, ...; per chunk all taps, 8 fmaf each;
    a shuffle-xor tree; then (c + acc) + bias and c - (x, y)."""
    B, H, W, cin = x.shape
    c8n = cin // 8
    xf, wf = x.float(), w.float()
    nb = [_neighbour(xf, t // 3 - 1, t % 3 - 1) for t in range(9)]
    lanes = []
    for lane in range(32):
        acc = [torch.zeros(B, H, W), torch.zeros(B, H, W)]
        for c8 in range(lane, c8n, 32):
            if c8 == drop_chunk:
                continue
            for t in range(9):
                for e in range(8):
                    ch = 8 * c8 + e
                    for o in range(2):
                        acc[o] = (nb[t][..., ch].double() * wf[o, ch, t // 3, t % 3].double() + acc[o].double()).float()
        lanes.append(acc)
    for off in (16, 8, 4, 2, 1):
        lanes = [[lanes[l][o] + lanes[l ^ off][o] for o in range(2)] for l in range(32)]
    a = torch.stack(lanes[0], -1)
    b = bias.float() * (2 if bias_twice else 1)
    c_out = (coords + a) + b
    return c_out, c_out - FR.grid_xy(B, H, W).float()


def head_simt_fp32(x, w, bias, coords):
    """The SIMT kernel's order: one fmaf chain over (tap, channel), + bias, + c, - (x, y)."""
    B, H, W, cin = x.shape
    xf, wf = x.float(), w.float()
    acc = [torch.zeros(B, H, W), torch.zeros(B, H, W)]
    for t in range(9):
        nb = _neighbour(xf, t // 3 - 1, t % 3 - 1)
        for ch in range(cin):
            for o in range(2):
                acc[o] = (nb[..., ch].double() * wf[o, ch, t // 3, t % 3].double() + acc[o].double()).float()
    v = torch.stack(acc, -1) + bias.float()
    c_out = coords + v
    return c_out, c_out - FR.grid_xy(B, H, W).float()


def taps_of(w, transposed=False):
    """engine._taps: the 3x3 -> 2 filter as 18 rows tap * 2 + o of a 1x1 layer (transposed: kx and ky swapped)."""
    return w.permute(3, 2, 0, 1).reshape(18, w.shape[1]) if transposed else w.permute(2, 3, 0, 1).reshape(18, w.shape[1])


def head_taps_fp32(x, w, bias, coords, transposed=False):
    """The tensor-core route: fp32 per-tap products (correctly rounded dot products), then flow_tap_gather_kernel's order."""
    B, H, W, cin = x.shape
    T = torch.einsum("bhwc,rc->bhwr", x.double(), taps_of(w, transposed).double()).float()  # [B,H,W,18]
    d = bias.float().expand(B, H, W, 2).clone()
    for t in range(9):
        d = d + _neighbour(T[..., 2 * t:2 * t + 2], t // 3 - 1, t % 3 - 1)  # zero outside the image: adds nothing
    c_out = coords + d
    return c_out, c_out - FR.grid_xy(B, H, W).float()


def test_engine_taps_layout():
    from ptlflow_b200.engine import _taps

    w = torch.randn(2, 16, 3, 3, generator=_gen(40))
    assert torch.equal(_taps(w).weight.view(18, 16), taps_of(w))
    assert not torch.equal(taps_of(w), taps_of(w, transposed=True))


@pytest.mark.parametrize("cin", [8, 64, 264])
@pytest.mark.parametrize("dtype", HALF, ids=["f16", "bf16"])
def test_flow_head_bound_admits_fp32_kernel_orders(cin, dtype):
    x, w, bias, coords = _head_operands(1, 3, 5, cin, dtype, cin)
    refs = _head_reference(x, w, bias, coords)
    routes = {"warp": head_warp_fp32, "taps": head_taps_fp32}
    if cin <= 64:
        routes["simt"] = head_simt_fp32
    for name, fn in routes.items():
        c_out, flow = fn(x, w, bias, coords)
        R.assert_within(c_out, *refs["coords"], what=f"{name} coords")
        R.assert_within(flow, *refs["out"], what=f"{name} flow")


@pytest.mark.parametrize("bug", ["bias_twice", "drop_chunk", "taps_transposed"])
def test_flow_head_bugs_rejected(bug):
    x, w, bias, coords = _head_operands(1, 4, 5, 64, torch.float16, 41)
    refs = _head_reference(x, w, bias, coords)
    if bug == "taps_transposed":
        _, flow = head_taps_fp32(x, w, bias, coords, transposed=True)
    else:
        _, flow = head_warp_fp32(x, w, bias, coords, **({"bias_twice": True} if bug == "bias_twice" else {"drop_chunk": 7}))
    assert R.max_ratio(flow, *refs["out"]) > 1.0


def test_flow_conv7x7_bound_admits_fmaf_chain():
    """The 7x7 motion-encoder conv of the fp32 flow (conv_flow7x7_kernel): bias first, then (ky, window column, kx) fmaf pairs."""
    g = _gen(50)
    flow = (torch.rand(1, 6, 9, 2, generator=g, dtype=torch.float64) * 2 - 1).mul(50).float()
    w = (torch.randn(16, 2, 7, 7, generator=g) * 98 ** -0.5).half()
    bias = torch.randn(16, generator=g) * 0.1
    acc, S, n = R.conv_terms([flow.double()], w.double(), bias.double())
    assert n == 99
    fp = F.pad(flow.permute(0, 3, 1, 2), (3, 3, 3, 3))
    got = bias.float().view(1, 16, 1, 1).expand(1, 16, 6, 9).clone()
    for ky in range(7):
        for kx in range(7):
            v = fp[:, :, ky:ky + 6, kx:kx + 9]
            for c in range(2):
                got = (w[:, c, ky, kx].double().view(1, 16, 1, 1) * v[:, c:c + 1].double() + got.double()).float()
    got = torch.relu(got).permute(0, 2, 3, 1).half()
    R.assert_within(got, *R.epilogue(R.RELU, acc, S, n, torch.float16)["out"], what="flow conv7x7")


# ------------------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------------------
def test_conv2d_flow_window_checked():
    """A FLOW output window without room for both components is refused before anything is launched (the pointers are never
    dereferenced)."""
    from helpers import lib as _lib

    L = _lib()
    lib = L.load()

    def params(stride, offset):
        p = L.ConvParams()
        p.src[0] = L.ConvSrc(16, 64, 64, 0, 0)
        p.nsrc, p.B, p.H, p.W, p.KH, p.KW = 1, 1, 4, 4, 3, 3
        p.Cout, p.Cout_pad, p.weight, p.bias, p.epilogue, p.scale = 2, 8, 16, 16, L.EPI_FLOW, 1.0
        p.out, p.out_stride, p.out_offset, p.coords, p.dtype = 16, stride, offset, 16, L.F16
        return p

    for stride, offset in ((2, 1), (8, 7), (1, 0), (4, -1)):
        assert lib.pfb_conv2d(C.byref(params(stride, offset)), None) == -1, (stride, offset)
        assert b"stride >= offset + 2" in lib.pfb_last_error()
