"""Conformance of the kernels that carry the fp32 flow against the float64 references of flow_reference.py and conv_reference.py,
element by element: the flow head's three routes (the warp kernel conv_cout2_flow_kernel, the SIMT FLOW epilogue, and the
per-tap GEMM + pfb_flow_tap_gather of the tensor-core loop), the convex upsamplers (8x, 4x, 2x in modes 0 and 1, CCMR's
handover), upflow8 / upflow2 / downflow, init_coords and the 7x7 motion-encoder convolution of the flow (conv_flow7x7_kernel).

Sources sit at an offset inside a wider pixel stride with NaN everywhere else; outputs are windows of sentinel-filled buffers
with spare elements behind them, which must keep the sentinel.  Operands on dyadic grids and one-hot masks make every fp32
step exact, so there the kernels must give the float64 (or exact fp32) result bit for bit.  With PFB_PARITY_REPORT set, every
case appends its max(err / bound) as one JSON line."""
import zlib

import pytest
import torch

import conv_reference as R
import flow_reference as FR
from helpers import _report, no_launch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HALF = [torch.float16, torch.bfloat16]
DT_IDS = {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32"}
IN_OFF = 8  # channel offset of the flow head's source inside its pixel stride (cin + 16)
OUT_STRIDE, OUT_OFF = 8, 2  # the flow head's output window
SPARE = 64  # sentinel elements behind every output


def _seed(*parts):
    return zlib.crc32("/".join(str(p) for p in parts).encode())


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _L():
    from ptlflow_b200 import _lib

    return _lib, _lib.load()


def _stream():
    from ptlflow_b200 import _lib

    return _lib.stream_ptr(torch.device(DEV))


def _sentinel(*shape):
    """(view of the given shape, whole buffer): fp32 sentinel with SPARE elements behind the view."""
    n = 1
    for s in shape:
        n *= s
    base = torch.full((n + SPARE,), FR.SENTINEL, dtype=torch.float32, device=DEV)
    return base[:n].view(*shape), base


def _spare_untouched(base, n, what):
    assert bool((base[n:] == FR.SENTINEL).all()), f"{what}: wrote past the end of its output"


def _coords(B, H, W, seed, amp=400.0):
    g = _gen(seed)
    return (FR.grid_xy(B, H, W, DEV) + (torch.rand(B, H, W, 2, generator=g, device=DEV, dtype=torch.float64) * 2 - 1) * amp).float()


# ------------------------------------------------------------------------------------------------------------------------------
# flow head
# ------------------------------------------------------------------------------------------------------------------------------
CIN = [8, 64, 128, 200, 256, 264, 512, 1024]  # 0, 1 and 2+ chunks per lane; 1024 is the warp kernel's limit
GRIDS = {"1x1": (1, 1, 1), "1xW": (1, 1, 37), "Hx1": (2, 29, 1), "ragged": (3, 7, 301), "bench": (8, 55, 128)}
HEAD_SHAPES = ([(g, c) for c in CIN for g in ("1x1", "ragged")] + [(g, c) for g in ("1xW", "Hx1") for c in (8, 264, 1024)]
               + [("bench", c) for c in (128, 256, 1024)])
ROUTES = [("warp", torch.float16), ("warp", torch.bfloat16), ("simt", torch.float16), ("simt", torch.bfloat16),
          ("simt", torch.float32), ("taps", torch.float16), ("taps", torch.bfloat16)]


class _Conv(torch.nn.Module):
    def __init__(self, weight, bias):
        super().__init__()
        self.weight, self.bias = weight, bias


def _head_operands(B, H, W, cin, dtype, seed, dyadic=False):
    """x [B,H,W,cin] (dtype), w [2,cin,3,3] fp32 (dtype-representable), bias fp32 [2], coords fp32 [B,H,W,2].  dyadic: small
    multiples of 1/4, 1/16 and 1/64, on which every fp32 partial sum of every route is exact."""
    g = _gen(seed)
    if dyadic:
        x = (torch.randint(-4, 5, (B, H, W, cin), generator=g, device=DEV) / 4.0).to(dtype)
        w = torch.randint(-4, 5, (2, cin, 3, 3), generator=g, device=DEV) / 16.0
        bias = torch.randint(-8, 9, (2,), generator=g, device=DEV) / 64.0
        coords = (FR.grid_xy(B, H, W, DEV) + torch.randint(-400 * 64, 400 * 64 + 1, (B, H, W, 2), generator=g, device=DEV) / 64.0).float()
        return x, w, bias.float(), coords
    x = torch.randn(B, H, W, cin, generator=g, device=DEV).to(dtype)
    w = torch.randn(2, cin, 3, 3, generator=g, device=DEV) * (9 * cin) ** -0.5
    bias = torch.randn(2, generator=g, device=DEV) * 0.1
    return x, w, bias, _coords(B, H, W, seed + 1)


def _wide_source(x, off=IN_OFF):
    """x inside a pixel stride of cin + 16 channels from ``off``, NaN elsewhere -> the conv2d source triple."""
    B, H, W, cin = x.shape
    t = torch.full((B, H, W, cin + 16), float("nan"), dtype=x.dtype, device=DEV)
    t[..., off:off + cin] = x
    return (t, cin, off)


def run_head(route, dtype, x, w, bias, coords):
    """One flow-head call on ``route`` -> (coords after the update, flow) as fp32 [B,H,W,2]; checks the sentinels."""
    from ptlflow_b200 import ops
    from ptlflow_b200.engine import _taps

    _lib, lib = _L()
    B, H, W, cin = x.shape
    src = _wide_source(x)
    c = coords.clone()
    if route == "taps":
        packed = ops.PackedConv([_taps(w)], dtype, DEV, src_channels=[cin])
        taps, _ = _sentinel(B, H, W, 32)
        before = taps.clone()
        ops.conv2d([src], packed, taps, _lib.EPI_LINEAR_F32, impl=2)
        R.assert_untouched(taps, before, 0, 18, what="taps")
        flow, base = _sentinel(B, H, W, 2)
        b = bias.float().contiguous()
        _lib.check(lib.pfb_flow_tap_gather(taps.data_ptr(), 32, b.data_ptr(), c.data_ptr(), flow.data_ptr(), B, H, W, _stream()),
                   "flow_tap_gather")
        torch.cuda.synchronize()
        _spare_untouched(base, flow.numel(), "flow_tap_gather")
        return c, flow
    packed = ops.PackedConv([_Conv(w, bias)], dtype, DEV, src_channels=[cin])
    out, base = _sentinel(B, H, W, OUT_STRIDE)
    before = out.clone()
    ops.conv2d([src], packed, out, _lib.EPI_FLOW, out_offset=OUT_OFF, coords=c, impl=2 if route == "warp" else 1)
    torch.cuda.synchronize()
    R.assert_untouched(out, before, OUT_OFF, OUT_OFF + 2, what=f"{route} output window")
    _spare_untouched(base, out.numel(), route)
    return c, out[..., OUT_OFF:OUT_OFF + 2]


def _head_refs(x, w, bias, coords, dtype):
    acc, S, n = R.conv_terms([x.double()], R.q(w, dtype), bias.double())
    assert n == 9 * x.shape[-1] + 1
    return R.epilogue(R.FLOW, acc, S, n, torch.float32, coords=coords.double())


@pytest.mark.parametrize("route,dtype", ROUTES, ids=[f"{r}-{DT_IDS[d]}" for r, d in ROUTES])
@pytest.mark.parametrize("grid,cin", HEAD_SHAPES, ids=[f"{g}-cin{c}" for g, c in HEAD_SHAPES])
def test_flow_head(grid, cin, route, dtype):
    B, H, W = GRIDS[grid]
    x, w, bias, coords = _head_operands(B, H, W, cin, dtype, _seed("head", grid, cin))
    refs = _head_refs(x, w, bias, coords, dtype)
    c, flow = run_head(route, dtype, x, w, bias, coords)
    what = f"flow head {route} {dtype} {grid} cin {cin}"
    worst = max(R.assert_within(c, *refs["coords"], what=what + " coords"), R.assert_within(flow, *refs["out"], what=what + " flow"))
    _report(test="flow_head", route=route, dtype=str(dtype), grid=grid, cin=cin, max_err_over_bound=worst)


DYADIC = [("ragged", 264), ("bench", 1024), ("1xW", 64), ("Hx1", 8)]


@pytest.mark.parametrize("route,dtype", ROUTES, ids=[f"{r}-{DT_IDS[d]}" for r, d in ROUTES])
@pytest.mark.parametrize("grid,cin", DYADIC, ids=[f"{g}-cin{c}" for g, c in DYADIC])
def test_flow_head_dyadic_exact(grid, cin, route, dtype):
    """Every fp32 partial sum is exact: coordinates and flow equal the float64 result bit for bit, twice."""
    B, H, W = GRIDS[grid]
    x, w, bias, coords = _head_operands(B, H, W, cin, dtype, _seed("dyadic", grid, cin), dyadic=True)
    refs = _head_refs(x, w, bias, coords, dtype)
    runs = [run_head(route, dtype, x, w, bias, coords) for _ in range(2)]
    for c, flow in runs:
        assert torch.equal(c.double(), refs["coords"][0]), f"{route} {dtype} coords"
        assert torch.equal(flow.double(), refs["out"][0]), f"{route} {dtype} flow"
    assert torch.equal(R.bits(runs[0][1].contiguous()), R.bits(runs[1][1].contiguous()))


DECLINED = ["cin12", "two_sources", "offset4"]


@pytest.mark.parametrize("dtype", HALF, ids=["f16", "bf16"])
@pytest.mark.parametrize("what", DECLINED)
def test_flow_head_warp_kernel_declines(what, dtype):
    """Shapes conv_cout2_supported declines: impl 2 raises before any launch; impl 0 computes them on the SIMT kernel."""
    from ptlflow_b200 import ops

    _lib, _ = _L()
    B, H, W = 2, 5, 9
    cin = 12 if what == "cin12" else 64
    x, w, bias, coords = _head_operands(B, H, W, cin, dtype, _seed("declined", what))
    if what == "two_sources":
        srcs, chans = [_wide_source(x[..., :32]), _wide_source(x[..., 32:])], [32, 32]
    else:
        srcs, chans = [_wide_source(x, 4 if what == "offset4" else IN_OFF)], [cin]
    packed = ops.PackedConv([_Conv(w, bias)], dtype, DEV, src_channels=chans)
    out, _ = _sentinel(B, H, W, OUT_STRIDE)
    before = out.clone()
    c = coords.clone()
    with no_launch():
        with pytest.raises(RuntimeError, match="wgmma path does not support"):
            ops.conv2d(srcs, packed, out, _lib.EPI_FLOW, out_offset=OUT_OFF, coords=c, impl=2)
    assert torch.equal(R.bits(out), R.bits(before)) and torch.equal(c, coords)
    ops.conv2d(srcs, packed, out, _lib.EPI_FLOW, out_offset=OUT_OFF, coords=c, impl=0)
    torch.cuda.synchronize()
    refs = _head_refs(x, w, bias, coords, dtype)
    R.assert_within(c, *refs["coords"], what=what + " coords")
    R.assert_within(out[..., OUT_OFF:OUT_OFF + 2], *refs["out"], what=what + " flow")
    R.assert_untouched(out, before, OUT_OFF, OUT_OFF + 2, what=what)


def test_flow_head_bad_window_refused_without_launch():
    from ptlflow_b200 import ops

    _lib, _ = _L()
    x, w, bias, coords = _head_operands(1, 4, 4, 64, torch.float16, 7)
    packed = ops.PackedConv([_Conv(w, bias)], torch.float16, DEV, src_channels=[64])
    out = torch.full((1, 4, 4, 4), FR.SENTINEL, device=DEV)
    for off in (3, -1):
        with no_launch():
            with pytest.raises(RuntimeError, match="stride >= offset"):
                ops.conv2d([_wide_source(x)], packed, out, _lib.EPI_FLOW, out_offset=off, coords=coords.clone(), impl=0)
    assert bool((out == FR.SENTINEL).all())


# ------------------------------------------------------------------------------------------------------------------------------
# convex upsamplers
# ------------------------------------------------------------------------------------------------------------------------------
KERNELS = {"x8": (8, 0), "x4": (4, 0), "x2": (2, 0), "x2_mode1": (2, 1), "handover": (2, 2)}
MASK_DTYPES = [torch.float16, torch.bfloat16, torch.float32]
SMALL = [(b, h, w) for b in (1, 3) for h, w in ((1, 1), (1, 9), (9, 1), (7, 11))]  # 77 pixels: a partial last block for every F


def _windows(FH, FW):
    """(out_hw, pad): the full grid, then a window 2 smaller (1 where the grid is 2 wide) at every legal pad."""
    dh, dw = min(2, FH - 1), min(2, FW - 1)
    return [((FH, FW), (0, 0))] + [((FH - dh, FW - dw), (pt, pl)) for pt in range(dh + 1) for pl in range(dw + 1)]


def run_convex(kernel, coords, mask, out_hw=None, pad=(0, 0)):
    """-> (output [B,2,oh,ow] (NCHW window; pixel-major modes permuted to NCHW), flow_small [B,2,H,W] or None)."""
    _lib, lib = _L()
    F_, mode = KERNELS[kernel]
    B, H, W, _ = coords.shape
    oh, ow = out_hw or (F_ * H, F_ * W)
    dt, s = _lib.dtype_code(mask.dtype), _stream()
    small, sbase = (None, None)
    if mode == 0:
        out, base = _sentinel(B, 2, oh, ow)
        if F_ in (8, 4):
            small, sbase = _sentinel(B, 2, H, W)
            fn = lib.pfb_convex_upsample if F_ == 8 else lib.pfb_convex_upsample4x
            rc = fn(coords.data_ptr(), mask.data_ptr(), out.data_ptr(), small.data_ptr(), B, H, W, oh, ow, pad[0], pad[1], dt, s)
        else:
            rc = lib.pfb_convex_upsample2x(coords.data_ptr(), mask.data_ptr(), out.data_ptr(), 0, B, H, W, oh, ow, pad[0], pad[1], dt, s)
    else:
        out, base = _sentinel(B, 2 * H, 2 * W, 2)
        if mode == 1:
            rc = lib.pfb_convex_upsample2x(coords.data_ptr(), mask.data_ptr(), out.data_ptr(), 1, B, H, W, 0, 0, 0, 0, dt, s)
        else:
            rc = lib.pfb_convex_handover2x(coords.data_ptr(), mask.data_ptr(), out.data_ptr(), B, H, W, dt, s)
    _lib.check(rc, kernel)
    torch.cuda.synchronize()
    _spare_untouched(base, out.numel(), kernel)
    if small is not None:
        _spare_untouched(sbase, small.numel(), kernel + " flow_small")
    return (out if mode == 0 else out.permute(0, 3, 1, 2)), small


def _check_flow_small(small, coords, what):
    B, H, W, _ = coords.shape
    want = (coords - FR.grid_xy(B, H, W, DEV).float()).permute(0, 3, 1, 2)
    assert torch.equal(R.bits(small.contiguous()), R.bits(want.contiguous())), what + " flow_small"


def _mask(B, H, W, F_, dtype, seed):
    return (torch.randn(B, H, W, 9 * F_ * F_, generator=_gen(seed), device=DEV) * 3.0).to(dtype)


@pytest.mark.parametrize("dtype", MASK_DTYPES, ids=["f16", "bf16", "f32"])
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("B,H,W", SMALL, ids=[f"b{b}-{h}x{w}" for b, h, w in SMALL])
def test_convex_upsample(B, H, W, kernel, dtype):
    F_, mode = KERNELS[kernel]
    sd = _seed("convex", kernel, B, H, W)
    coords = _coords(B, H, W, sd)
    mask = _mask(B, H, W, F_, dtype, sd + 1)
    ref, bound = FR.convex(coords, mask, F_, mode)
    worst = 0.0
    for out_hw, pad in (_windows(F_ * H, F_ * W) if mode == 0 else [(None, (0, 0))]):
        got, small = run_convex(kernel, coords, mask, out_hw, pad)
        oh, ow = got.shape[-2:]
        win = lambda t: t[:, :, pad[0]:pad[0] + oh, pad[1]:pad[1] + ow]  # noqa: E731
        worst = max(worst, FR.assert_within(got, win(ref), win(bound), f"{kernel} {dtype} {out_hw} at {pad}"))
        if small is not None:
            _check_flow_small(small, coords, kernel)
    _report(test="convex_upsample", kernel=kernel, dtype=str(dtype), shape=[B, H, W], max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", MASK_DTYPES, ids=["f16", "bf16", "f32"])
def test_convex_upsample_bench_shape(dtype):
    """The bench's 8 x 55 x 128 grid, 8x, cropped to 436 x 1024 at pad (2, 0)."""
    B, H, W = 8, 55, 128
    coords = _coords(B, H, W, 91)
    mask = _mask(B, H, W, 8, dtype, 92)
    ref, bound = FR.convex(coords, mask, 8)
    got, small = run_convex("x8", coords, mask, (436, 1024), (2, 0))
    worst = FR.assert_within(got, ref[:, :, 2:438], bound[:, :, 2:438], f"x8 bench {dtype}")
    _check_flow_small(small, coords, "x8 bench")
    _report(test="convex_upsample", kernel="x8", dtype=str(dtype), shape=[B, H, W], max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", MASK_DTYPES, ids=["f16", "bf16", "f32"])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_convex_upsample_onehot_exact(kernel, dtype):
    """One logit at 0 and eight at -120 (expf of -120 is exactly 0 in fp32): the kernel is a gather and gives F * fp32(c - g)
    of the dominant tap (0 outside the image; mode 2 plus the fine grid) bit for bit.  The dominant tap runs over all 9 taps
    at every sub-pixel."""
    F_, mode = KERNELS[kernel]
    B, H, W = 2, 5, 6
    coords = _coords(B, H, W, _seed("onehot", kernel))
    FF = F_ * F_
    for k in range(9):
        tap = (torch.arange(FF, device=DEV).view(1, 1, 1, F_, F_) + torch.arange(H * W, device=DEV).view(1, H, W, 1, 1) + k) % 9
        tap = tap.expand(B, H, W, F_, F_)
        mask = torch.full((B, H, W, 9, FF), -120.0, device=DEV)
        mask.scatter_(3, tap.reshape(B, H, W, 1, FF), 0.0)
        mask = mask.view(B, H, W, 9 * FF).to(dtype)
        got, _ = run_convex(kernel, coords, mask)
        want = FR.onehot_expected(coords, tap, F_, mode)
        assert torch.equal(R.bits(got.contiguous()), R.bits(want.contiguous())), f"{kernel} {dtype} dominant tap shift {k}"


# ------------------------------------------------------------------------------------------------------------------------------
# upflow8, upflow2, downflow, init_coords
# ------------------------------------------------------------------------------------------------------------------------------
RESAMPLE = SMALL + [(8, 55, 128)]


@pytest.mark.parametrize("B,H,W", RESAMPLE, ids=[f"b{b}-{h}x{w}" for b, h, w in RESAMPLE])
def test_upflow8(B, H, W):
    _lib, lib = _L()
    coords = _coords(B, H, W, _seed("upflow8", B, H, W))
    wins = [((436, 1024), (2, 0))] if (H, W) == (55, 128) else _windows(8 * H, 8 * W)
    worst = 0.0
    for (oh, ow), pad in wins:
        out, base = _sentinel(B, 2, oh, ow)
        small, sbase = _sentinel(B, 2, H, W)
        _lib.check(lib.pfb_upflow8(coords.data_ptr(), out.data_ptr(), small.data_ptr(), B, H, W, oh, ow, pad[0], pad[1], _stream()), "upflow8")
        torch.cuda.synchronize()
        _spare_untouched(base, out.numel(), "upflow8")
        _spare_untouched(sbase, small.numel(), "upflow8 flow_small")
        worst = max(worst, FR.assert_within(out, *FR.upflow(coords, 8, (oh, ow), pad), f"upflow8 {(oh, ow)} at {pad}"))
        _check_flow_small(small, coords, "upflow8")
    _report(test="upflow8", shape=[B, H, W], max_err_over_bound=worst)


def _flow(B, H, W, seed, amp=400.0):
    return ((torch.rand(B, 2, H, W, generator=_gen(seed), device=DEV, dtype=torch.float64) * 2 - 1) * amp).float()


@pytest.mark.parametrize("B,H,W", RESAMPLE, ids=[f"b{b}-{h}x{w}" for b, h, w in RESAMPLE])
def test_upflow2(B, H, W):
    _lib, lib = _L()
    flow = _flow(B, H, W, _seed("upflow2", B, H, W))
    worst = 0.0
    for (oh, ow), pad in _windows(2 * H, 2 * W):
        out, base = _sentinel(B, 2, oh, ow)
        _lib.check(lib.pfb_upflow2(flow.data_ptr(), out.data_ptr(), B, H, W, oh, ow, pad[0], pad[1], _stream()), "upflow2")
        torch.cuda.synchronize()
        _spare_untouched(base, out.numel(), "upflow2")
        worst = max(worst, FR.assert_within(out, *FR.upflow2(flow, (oh, ow), pad), f"upflow2 {(oh, ow)} at {pad}"))
    _report(test="upflow2", shape=[B, H, W], max_err_over_bound=worst)


DOWN = [((1, 1, 1), (1, 1)), ((3, 7, 11), (1, 1)), ((3, 7, 11), (3, 4)), ((1, 1, 9), (1, 3)), ((3, 9, 1), (4, 1)),
        ((2, 55, 128), (3, 8)), ((1, 7, 11), (7, 11)), ((2, 3, 5), (7, 9))]


@pytest.mark.parametrize("shape,out_hw", DOWN, ids=[f"{s[1]}x{s[2]}-to-{o[0]}x{o[1]}" for s, o in DOWN])
def test_downflow(shape, out_hw):
    _lib, lib = _L()
    B, H, W = shape
    flow = _flow(B, H, W, _seed("downflow", shape, out_hw))
    out, base = _sentinel(B, 2, *out_hw)
    _lib.check(lib.pfb_downflow(flow.data_ptr(), out.data_ptr(), B, H, W, out_hw[0], out_hw[1], _stream()), "downflow")
    torch.cuda.synchronize()
    _spare_untouched(base, out.numel(), "downflow")
    worst = FR.assert_within(out, *FR.downflow(flow, out_hw), f"downflow {shape} -> {out_hw}")
    _report(test="downflow", shape=list(shape), out_hw=list(out_hw), max_err_over_bound=worst)


@pytest.mark.parametrize("B,H,W", RESAMPLE, ids=[f"b{b}-{h}x{w}" for b, h, w in RESAMPLE])
def test_init_coords(B, H, W):
    """The grid, plus flow_init in one fp32 addition: bit for bit."""
    _lib, lib = _L()
    grid = FR.grid_xy(B, H, W, DEV).float()
    fi = _flow(B, H, W, _seed("init", B, H, W))
    for flow_init in (None, fi):
        c, base = _sentinel(B, H, W, 2)
        _lib.check(lib.pfb_init_coords(c.data_ptr(), flow_init.data_ptr() if flow_init is not None else None, B, H, W, _stream()),
                   "init_coords")
        torch.cuda.synchronize()
        _spare_untouched(base, c.numel(), "init_coords")
        want = grid if flow_init is None else grid + flow_init.permute(0, 2, 3, 1)
        assert torch.equal(R.bits(c), R.bits(want.contiguous()))


# ------------------------------------------------------------------------------------------------------------------------------
# 7x7 convolution of the flow (motion encoder convf1)
# ------------------------------------------------------------------------------------------------------------------------------
F7_GRIDS = [(1, 55, 128), (2, 3, 256), (1, 5, 300), (1, 1, 1)]  # W % 128 == 0: the <1,128> row tile; otherwise <8,16>


@pytest.mark.parametrize("dtype", HALF, ids=["f16", "bf16"])
@pytest.mark.parametrize("cout", [64, 128, 192])
@pytest.mark.parametrize("B,H,W", F7_GRIDS, ids=[f"b{b}-{h}x{w}" for b, h, w in F7_GRIDS])
def test_flow_conv7x7(B, H, W, cout, dtype):
    """impl 2 reaches conv_flow7x7_kernel or raises; auto selection (impl 0) gives the same bits."""
    from ptlflow_b200 import ops

    _lib, _ = _L()
    sd = _seed("f7", B, H, W, cout)
    g = _gen(sd)
    flow = _flow(B, H, W, sd + 1, amp=50.0).permute(0, 2, 3, 1).contiguous()
    w = torch.randn(cout, 2, 7, 7, generator=g, device=DEV) * 98 ** -0.5
    bias = torch.randn(cout, generator=g, device=DEV) * 0.1
    packed = ops.PackedConv([_Conv(w, bias)], dtype, DEV)
    off, stride = 8, cout + 16
    outs = []
    for impl in (2, 0):
        out = torch.full((B, H, W, stride), FR.SENTINEL, dtype=dtype, device=DEV)
        before = out.clone()
        ops.conv2d([flow], packed, out, _lib.EPI_RELU, out_offset=off, impl=impl)
        torch.cuda.synchronize()
        R.assert_untouched(out, before, off, off + cout, what=f"flow conv7x7 impl {impl}")
        outs.append(out)
    acc, S, n = R.conv_terms([flow.double()], R.q(w, dtype), bias.double())
    assert n == 99
    worst = R.assert_within(outs[0][..., off:off + cout], *R.epilogue(R.RELU, acc, S, n, dtype)["out"], what=f"flow conv7x7 {dtype}")
    assert torch.equal(R.bits(outs[0]), R.bits(outs[1]))
    _report(test="flow_conv7x7", shape=[B, H, W], cout=cout, dtype=str(dtype), max_err_over_bound=worst)
