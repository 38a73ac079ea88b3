"""The float64 correlation reference and its per-element bounds (corr_reference.py) on the CPU.

* It agrees with the fp32 oracle (oracle/raft_oracle.py) and with the vectors the real reference wrote
  (tests/golden/op_corr_lookup.npz, op_alt_corr.npz).
* A torch emulation of each kernel's rounding scheme (fp32 accumulation in another order, storage rounding where the kernel
  rounds, the tensor-core accumulator dump) stays inside its bound.
* Each of a set of plausible kernel bugs, planted into an emulation, falls outside the bound.
* otf_plan gives the tensor-core on-the-fly kernel's bands and flags on hand-built tiles."""
import math

import numpy as np
import pytest
import torch

import corr_reference as R
from helpers import load_golden
from oracle import raft_oracle as O
from oracle import synth

DTYPES = [torch.float16, torch.bfloat16]
K4 = 9  # window side at radius 4


def _gen(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g, dtype=torch.float64) * scale


def _rt(x, dtype):
    """float32 x rounded to the storage type, back as float32."""
    return x.to(dtype).float()


# ---------------------------------------------------------------------------------------------------------------------
# emulations of the kernels' rounding (fp32 on the CPU)
# ---------------------------------------------------------------------------------------------------------------------
def emu_dots(f1, f2):
    """Raw dots [B*H1*W1, H2, W2] in fp32, accumulated over 16-channel blocks in reverse order (not the reference's)."""
    B, H1, W1, C = f1.shape
    H2, W2 = f2.shape[1:3]
    a = f1.float().reshape(B, H1 * W1, C)
    b = f2.float().reshape(B, H2 * W2, C)
    acc = torch.zeros(B, H1 * W1, H2 * W2, dtype=torch.float32)
    for k in reversed(range(0, C, 16)):
        acc = acc + torch.bmm(a[..., k:k + 16], b[..., k:k + 16].transpose(1, 2))
    return acc.reshape(B * H1 * W1, H2, W2)


def emu_volume(f1, f2, scale, dtype, mutant=None):
    s = torch.tensor(scale, dtype=torch.float32)
    v = emu_dots(f1, f2) * s
    if mutant == "scale_twice":
        v = v * s
    return _rt(v, dtype)


def _pool_f32(x, l, mutant=None):
    """fp32 sums of 2^l x 2^l blocks (tree of pair sums), floor sizes; mutant: the row pairs shifted by one."""
    for _ in range(l):
        h, w = x.shape[-2] // 2, x.shape[-1] // 2
        if mutant == "wrong_row_pair":
            xs = torch.cat([x, x[..., -1:, :]], -2)[..., 1:2 * h + 1, :2 * w]
        else:
            xs = x[..., :2 * h, :2 * w]
        x = (xs[..., 0::2, 0::2] + xs[..., 0::2, 1::2]) + (xs[..., 1::2, 0::2] + xs[..., 1::2, 1::2])
    return x


def emu_pyramid_once(f1, f2, scale, dtype, levels, mutant=None):
    acc = emu_dots(f1, f2)
    out = []
    for l in range(levels):
        s = torch.tensor(scale * 4.0 ** -l, dtype=torch.float32)
        out.append(_rt(_pool_f32(acc, l, mutant if l else None) * s, dtype))
    return out


def emu_pool2x2(x, dtype):
    """avg_pool2x2 on stored x [..., H, W] (fp32): one fp32 sum of four, times 0.25, one rounding."""
    h, w = x.shape[-2] // 2, x.shape[-1] // 2
    x = x[..., :2 * h, :2 * w]
    s = ((x[..., 0::2, 0::2] + x[..., 0::2, 1::2]) + x[..., 1::2, 0::2]) + x[..., 1::2, 1::2]
    return _rt(0.25 * s, dtype)


def emu_pyramid_rerounded(f1, f2, scale, dtype, levels):
    out = [emu_volume(f1, f2, scale, dtype)]
    for _ in range(1, levels):
        out.append(emu_pool2x2(out[-1], dtype))
    return out


def _weights32(coords, l, mutant=None):
    """Window origin and fp32 tap weights as the lookup kernels compute them (mutant: floor taken before the level scale)."""
    c = coords.float()
    if mutant == "floor_before_scale":
        c = torch.floor(c)
    c = c * (2.0 ** -l)
    x, y = c[:, 0], c[:, 1]
    fin = (x.abs() < 1e7) & (y.abs() < 1e7)
    xf = torch.where(fin, torch.floor(x), torch.full_like(x, -1e6))
    yf = torch.where(fin, torch.floor(y), torch.full_like(y, -1e6))
    fx = torch.where(fin, x - xf, torch.zeros_like(x))
    fy = torch.where(fin, y - yf, torch.zeros_like(y))
    one = torch.ones_like(fx)
    w = [(one - fx) * (one - fy), fx * (one - fy), (one - fx) * fy, fx * fy]
    if mutant == "swap_w10_w01":
        w[1], w[2] = w[2], w[1]
    return xf.long() - 4, yf.long() - 4, w


def _blend(taps, w, mutant=None):
    """taps: four [Q, K*K] fp32 tap values, w: four [Q] fp32 weights -> [Q, K*K] fp32 in the kernels' order."""
    v = w[0][:, None] * taps[0] + w[1][:, None] * taps[1] + w[2][:, None] * taps[2] + w[3][:, None] * taps[3]
    if mutant == "y_major":
        v = v.view(-1, K4, K4).transpose(1, 2).reshape(-1, K4 * K4)
    return v


def emu_lookup(levels32, coords, dtype, mutant=None):
    """Lookup at radius 4 from dense stored levels (fp32 [Q, h, w])."""
    out = []
    for l, V in enumerate(levels32):
        x0, y0, w = _weights32(coords, l, mutant)
        taps = [R.gather_window(V, x0, y0, K4, dx, dy) for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1))]
        if mutant == "tap_shifted":  # tap w11 read one column further right
            taps[3] = R.gather_window(V, x0, y0, K4, 2, 1)
        out.append(_blend(taps, w, mutant))
    return _rt(torch.cat(out, 1), dtype)


def _t84_taps(tiled, h, w, x0, y0, dx, dy, tiles_x, mask_pad):
    """The tiled kernel's tap reads: rows < h, tile columns < tiles_x, pad columns masked unless mask_pad is False."""
    Q = tiled.shape[0]
    k = torch.arange(K4)
    xi = (x0.view(Q, 1, 1) + k.view(1, K4, 1) + dx).expand(Q, K4, K4)
    yi = (y0.view(Q, 1, 1) + k.view(1, 1, K4) + dy).expand(Q, K4, K4)
    ok = (yi >= 0) & (yi < h) & (xi >= 0) & ((xi >> 3) < (w + 7) // 8)
    if mask_pad:
        ok &= xi < w
    yc, xc = yi.clamp(0, h - 1), xi.clamp(0, (w + 7) // 8 * 8 - 1)
    off = ((yc >> 2) * tiles_x + (xc >> 3)) * 32 + (yc & 3) * 8 + (xc & 7)
    off = off.clamp(0, tiled.shape[1] - 1).reshape(Q, -1)
    v = torch.gather(tiled, 1, off)
    return torch.where(ok.reshape(Q, -1), v, torch.zeros_like(v))


def emu_lookup_tiled(tiled32, hw, coords, dtype, mutant=None):
    out = []
    for l, (T, (h, w)) in enumerate(zip(tiled32, hw)):
        x0, y0, wt = _weights32(coords, l)
        tiles_x = (hw[0][1] + 7) // 8 if (mutant == "tiles_x_of_level0" and l) else (w + 7) // 8
        taps = [_t84_taps(T, h, w, x0, y0, dx, dy, tiles_x, mutant != "pad_unmasked") for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1))]
        out.append(_blend(taps, wt))
    return _rt(torch.cat(out, 1), dtype)


def emu_onthefly(f1, f2_levels, coords, scale, dtype, tensor_cores, mutant=None):
    s = torch.tensor(scale, dtype=torch.float32)
    out = []
    for l, f2 in enumerate(f2_levels):
        d = emu_dots(f1, f2)
        if tensor_cores:  # the accumulator dump: scaled, rounded to storage (the old kernel rounded the raw dot)
            d = _rt(d, dtype) * s if mutant == "dump_before_scale" else _rt(d * s, dtype)
        x0, y0, w = _weights32(coords, l)
        if not tensor_cores:
            w = [wi * s for wi in w]
        taps = [R.gather_window(d, x0, y0, K4, dx, dy) for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1))]
        out.append(_blend(taps, w))
    return _rt(torch.cat(out, 1), dtype)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _feats(dtype, B=1, H=9, W=13, C=64, seed=0, H2=None, W2=None, mag=1.0):
    f1 = R.q(_gen((B, H, W, C), seed, mag), dtype)
    f2 = R.q(_gen((B, H2 or H, W2 or W, C), seed + 1, mag), dtype)
    return f1, f2


def _coords(Q, H, W, seed, sigma=3.0):
    """Query coordinates [Q, 2] float32 around the grid, with edge cases: integers, x = W - 1, -1e-7, -40, NaN, inf, values
    either side of 1e7 at every level, and windows starting at every tile column."""
    g = torch.Generator().manual_seed(seed)
    c = torch.stack([torch.rand(Q, generator=g) * W, torch.rand(Q, generator=g) * H], 1) + sigma * torch.randn(Q, 2, generator=g)
    special = [(3.0, 2.0), (W - 1.0, H / 2), (-1e-7, 1.0), (-40.0, 2.0), (float("nan"), 1.0), (1.0, float("inf")),
               (float("-inf"), 0.0), (W / 2, -1e-7), (W - 1.0, H - 1.0)]
    for l in range(4):
        t = 1e7 * 2.0 ** l
        below = float(np.nextafter(np.float32(t), np.float32(0)))
        special += [(below, 1.0), (t, 1.0), (-t, 1.0), (1.0, -below)]
    special += [(8.0 * (k // 8) + k % 8 + 4 + 0.25, 2.5) for k in range(8)]  # window origin at tile column 0..7
    for i, (x, y) in enumerate(special[:Q]):
        c[i, 0], c[i, 1] = float(x), float(y)
    return c.float()


# ---------------------------------------------------------------------------------------------------------------------
# agreement with the existing references
# ---------------------------------------------------------------------------------------------------------------------
def _golden_inputs(recipe):
    b, c, h, w = recipe["b"], recipe["c"], recipe["h"], recipe["w"]
    f1 = torch.from_numpy(synth.synth_normal("ops/fmap1", (b, c, h, w), recipe["seed"]))
    f2 = torch.from_numpy(synth.synth_normal("ops/fmap2", (b, c, h, w), recipe["seed"]))
    return f1, f2


def _dense_pyramid(f1, f2, levels):
    """float64 reference pyramid from NCHW features."""
    ref0, _ = R.volume(f1.permute(0, 2, 3, 1), f2.permute(0, 2, 3, 1), f1.shape[1] ** -0.5)
    return [R.pool(ref0, l) for l in range(levels)]


def _nchw(look, B, H, W):
    return look.view(B, H, W, -1).permute(0, 3, 1, 2)


def _pm_coords(coords):
    return coords.permute(0, 2, 3, 1).reshape(-1, 2).float()


def test_agrees_with_oracle_volume_pyramid_lookup():
    f1, f2 = _gen((2, 48, 7, 11), 1).float(), _gen((2, 48, 7, 11), 2).float()
    pyr_o = O.corr_pyramid(O.corr_volume(f1, f2), 3)
    pyr_r = _dense_pyramid(f1.double(), f2.double(), 3)
    for po, pr in zip(pyr_o, pyr_r):
        assert (po[:, 0].double() - pr).abs().max() < 1e-5
    coords = O.coords_grid(2, 7, 11) + 2.5 * torch.randn(2, 2, 7, 11, generator=torch.Generator().manual_seed(3))
    look_o = O.corr_lookup(pyr_o, coords, 3)
    look_r, _ = R.lookup(pyr_r, _pm_coords(coords), 3, torch.float32)
    assert (look_o.double() - _nchw(look_r, 2, 7, 11)).abs().max() < 2e-5
    # on the fly: level l correlates fmap1 with fmap2 pooled l times
    f2p = [f2.double().permute(0, 2, 3, 1)]
    for _ in range(2):
        f2p.append(R.avg_pool2x2(f2p[-1], torch.float32)[0])
    alt_o = O.alt_corr_lookup(f1, f2, coords, 3, 3)
    alt_r, _ = R.onthefly(f1.double().permute(0, 2, 3, 1), f2p, _pm_coords(coords), 3, 48 ** -0.5, torch.float32, False)
    assert (alt_o.double() - _nchw(alt_r, 2, 7, 11)).abs().max() < 2e-5


def test_agrees_with_reference_vectors():
    recipe, g = load_golden("op_corr_lookup")
    f1, f2 = _golden_inputs(recipe)
    B, H, W, L, r = recipe["b"], recipe["h"], recipe["w"], recipe["levels"], recipe["radius"]
    pyr = _dense_pyramid(f1.double(), f2.double(), L)
    assert np.abs(pyr[3].numpy() - g["level3"][:, 0]).max() < 1e-5
    look, _ = R.lookup(pyr, _pm_coords(torch.from_numpy(g["coords"])), r, torch.float32)
    assert np.abs(_nchw(look, B, H, W).numpy() - g["lookup"]).max() < 2e-5

    recipe, g = load_golden("op_alt_corr")
    f1, f2 = _golden_inputs(recipe)
    f2p = [f2.double().permute(0, 2, 3, 1)]
    for _ in range(recipe["levels"] - 1):
        f2p.append(R.avg_pool2x2(f2p[-1], torch.float32)[0])
    alt, _ = R.onthefly(f1.double().permute(0, 2, 3, 1), f2p, _pm_coords(torch.from_numpy(g["coords"])), recipe["radius"],
                        recipe["c"] ** -0.5, torch.float32, False)
    assert np.abs(_nchw(alt, recipe["b"], recipe["h"], recipe["w"]).numpy() - g["lookup"]).max() < 5e-5


def test_t84_restatement():
    """The tiled address formula: element (y, x) at ((y >> 2) * tiles_x + (x >> 3)) * 32 + (y & 3) * 8 + (x & 7)."""
    h, w = 6, 11  # tiles_y 2, tiles_x 2
    dense = torch.arange(h * w, dtype=torch.float64).view(1, h, w)
    t = R.t84_write(dense, pad_value=-1.0)
    assert t.shape == (1, 2 * 2 * 32)
    assert t[0, 0] == 0 and t[0, 8] == w and t[0, 32] == 8 and t[0, 64] == 4 * w
    assert t[0, 32 + 3] == -1.0  # column 11 of row 0: a pad column
    assert torch.equal(R.t84_read(t, h, w), dense)
    assert int(R.t84_pad_mask(h, w).sum()) == 2 * 2 * 32 - h * w


# ---------------------------------------------------------------------------------------------------------------------
# emulations stay inside the bounds
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES + [torch.float32], ids=["float16", "bfloat16", "float32"])
@pytest.mark.parametrize("C", [64, 192])
def test_volume_emulations_inside(dtype, C):
    f1, f2 = _feats(dtype, B=2, H=9, W=21, C=C, seed=C)
    s = C ** -0.5
    ref0, S = R.volume(f1, f2, s)
    for l, ((r, b), got) in enumerate(zip(R.pyramid_rerounded(ref0, S, C, s, dtype, 3), emu_pyramid_rerounded(f1, f2, s, dtype, 3))):
        assert R.assert_within(got, r, b, f"rerounded level {l}") <= 1.0
    if dtype != torch.float32:
        for l, ((r, b), got) in enumerate(zip(R.pyramid_once(ref0, S, C, s, dtype, 3), emu_pyramid_once(f1, f2, s, dtype, 3))):
            assert R.assert_within(got, r, b, f"once level {l}") <= 1.0


@pytest.mark.parametrize("dtype", DTYPES + [torch.float32], ids=["float16", "bfloat16", "float32"])
def test_pool_and_lookup_emulations_inside(dtype):
    x = R.q(_gen((2, 7, 9, 16), 5), dtype)
    ref, bound = R.avg_pool2x2(x, dtype)
    got = emu_pool2x2(x.float().movedim(-1, 1), dtype).movedim(1, -1)
    R.assert_within(got, ref, bound, "avg_pool2x2")
    Q, hw = 96, [(11, 21), (5, 10), (2, 5), (1, 2)]
    levels = [R.q(_gen((Q, h, w), 10 + l), dtype) for l, (h, w) in enumerate(hw)]
    coords = _coords(Q, 11, 21, 7)
    ref, bound = R.lookup(levels, coords, 4, dtype)
    R.assert_within(emu_lookup([v.float() for v in levels], coords, dtype), ref, bound, "lookup")
    if dtype != torch.float32:
        tiled = [R.t84_write(v.float(), 1000.0) for v in levels]
        R.assert_within(emu_lookup_tiled(tiled, hw, coords, dtype), ref, bound, "tiled lookup")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("tensor_cores", [False, True], ids=["simt", "tc"])
@pytest.mark.parametrize("C,scale", [(64, 0.125), (128, 128 ** -0.5), (128, 96 ** -0.5)])
def test_onthefly_emulations_inside(dtype, tensor_cores, C, scale):
    B, H, W = 1, 9, 21
    f1, f2 = _feats(dtype, B=B, H=H, W=W, C=C, seed=C)
    f2p = [f2]
    for _ in range(2):
        f2p.append(R.q(R.avg_pool2x2(f2p[-1], dtype)[0], dtype))
    coords = _coords(B * H * W, H, W, 9)
    ref, bound = R.onthefly(f1, f2p, coords, 4, scale, dtype, tensor_cores)
    R.assert_within(emu_onthefly(f1, f2p, coords, scale, dtype, tensor_cores), ref, bound, "on the fly")


def test_onthefly_f16_dot_overflow():
    """|a.b| > 65504 with a scaled correlation well inside f16: rounding the raw dot to f16 before the scale gives inf; the
    scaled dump stays finite and inside the bound."""
    dtype, C = torch.float16, 256
    f1, _ = _feats(dtype, B=1, H=4, W=9, C=C, seed=3, mag=20.0)
    f2 = f1.clone()  # the window centre tap: a.a = |a|^2 ~ 256 * 400, above 65504
    coords = _grid(1, 4, 9).reshape(-1, 2)
    ref, bound = R.onthefly(f1, [f2], coords, 4, C ** -0.5, dtype, True)
    assert R.ratio(emu_onthefly(f1, [f2], coords, C ** -0.5, dtype, True), ref, bound).max() <= 1.0
    assert R.ratio(emu_onthefly(f1, [f2], coords, C ** -0.5, dtype, True, "dump_before_scale"), ref, bound).max() > 1.0


# ---------------------------------------------------------------------------------------------------------------------
# mutants fall outside
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mutant", ["tap_shifted", "swap_w10_w01", "y_major", "floor_before_scale"])
def test_lookup_mutants_rejected(mutant, dtype):
    Q, hw = 96, [(11, 21), (5, 10), (2, 5)]
    levels = [R.q(_gen((Q, h, w), 20 + l), dtype) for l, (h, w) in enumerate(hw)]
    coords = _coords(Q, 11, 21, 8)
    ref, bound = R.lookup(levels, coords, 4, dtype)
    got = emu_lookup([v.float() for v in levels], coords, dtype, mutant)
    assert R.ratio(got, ref, bound).max() > 1.0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mutant", ["pad_unmasked", "tiles_x_of_level0"])
def test_tiled_lookup_mutants_rejected(mutant, dtype):
    Q, hw = 96, [(11, 21), (5, 10), (2, 5)]
    levels = [R.q(_gen((Q, h, w), 30 + l), dtype) for l, (h, w) in enumerate(hw)]
    coords = _coords(Q, 11, 21, 9)
    coords[40:60, 0] = 20.5  # windows that reach the pad columns of level 0 (w = 21: columns 21..23)
    ref, bound = R.lookup(levels, coords, 4, dtype)
    tiled = [R.t84_write(v.float(), 1000.0) for v in levels]
    assert R.ratio(emu_lookup_tiled(tiled, hw, coords, dtype, mutant), ref, bound).max() > 1.0


@pytest.mark.parametrize("dtype", DTYPES)
def test_volume_mutants_rejected(dtype):
    C = 64
    f1, f2 = _feats(dtype, B=1, H=9, W=21, C=C, seed=40)
    s = C ** -0.5
    ref0, S = R.volume(f1, f2, s)
    assert R.ratio(emu_volume(f1, f2, s, dtype, "scale_twice"), ref0, R.volume_bound(ref0, S, C, s, dtype)).max() > 1.0
    once = R.pyramid_once(ref0, S, C, s, dtype, 3)
    bad = emu_pyramid_once(f1, f2, s, dtype, 3, "wrong_row_pair")
    for l in (1, 2):
        assert R.ratio(bad[l], *once[l]).max() > 1.0


# ---------------------------------------------------------------------------------------------------------------------
# otf_plan on hand-built tiles
# ---------------------------------------------------------------------------------------------------------------------
def _grid(B, H, W):
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    return torch.stack([xs, ys], -1)[None].repeat(B, 1, 1, 1)


def test_otf_plan_smooth_tile():
    c = _grid(1, 8, 16)
    nb, bx, by, flags = R.otf_plan(c, 8, 16, 2)
    # level 0: windows from y0 = -4 (row 0) to 3 (row 7): 17 region rows, 3 bands; level 1: y0 -4..-1, 2 bands
    assert nb.tolist() == [3, 2] and bx.tolist() == [-4, -4] and by.tolist() == [-4, -4]
    assert not flags.any()


def test_otf_plan_rough_flow_reaches_eight_bands():
    H, W = 128, 16
    c = _grid(1, H, W)
    c[0, :8, :, 1] = (16 * torch.arange(8, dtype=torch.float32) + 4).view(8, 1)  # tile 0: rows 16 apart, y0 = 0, 16, .., 112
    nb, bx, by, flags = R.otf_plan(c, H, W, 1)
    assert nb[0] == 8 and by[0] == 0
    # 8 bands serve region rows 0..56: windows with ryo + 9 <= 56, i.e. y0 <= 47 (rows 0..2 of the tile)
    assert flags[0, :3].sum() == 0 and bool(flags[0, 3:8].all())
    assert not flags[0, 8:].any()


def test_otf_plan_window_right_of_anchor():
    c = _grid(1, 8, 64)
    c[0, :, :16, 0] = 20.0
    c[0, 3, 5, 0] = 20.0 + 23  # cxo = 23: 23 + 10 > 32
    c[0, 4, 6, 0] = 20.0 + 22  # cxo = 22: the window's last column is region column 31
    _, bx, _, flags = R.otf_plan(c, 8, 64, 1)
    assert bx[0] == 16
    assert flags[0, 3, 5] and not flags[0, 4, 6]
    assert int(flags.sum()) == 1


def test_otf_plan_dead_tiles_and_negative_anchor():
    c = _grid(1, 16, 32)
    c[0, :8, :16] = float("nan")           # tile (0, 0): no live query: no band, anchor (0, 0)
    c[0, 8:, :16] = -30.0                  # tile (1, 0): windows wholly left of / above the map: dead too
    c[0, :8, 16:, 0] -= 20.0               # tile (0, 1): x0 from -8 to 7 with the window still overlapping
    nb, bx, by, flags = R.otf_plan(c, 16, 32, 1)
    assert nb.tolist()[:3] == [0, 3, 0] and bx.tolist()[:3] == [0, -8, 0] and by.tolist()[:3] == [0, -4, 0]
    assert bx[3] == 12 and by[3] == 4 and not flags.any()
