"""Float64 reference of the correlation path (volume, pooled pyramid, lookup, on-the-fly lookup, feature pooling) and an
error bound per output element (TEST INFRASTRUCTURE, like conv_reference.py).  test_gpu_corr_conformance.py compares the
kernels of csrc/corr.cu, corr_umma.cu, corr_tiled.cu and corr_onthefly_umma.cu with it; test_corr_reference.py shows on
the CPU that rounding emulations stay inside the bounds and that plausible kernel bugs fall outside them.

Notation.  a and b are the features as stored (already rounded to the storage type), in float64; s is the scale; for each
(query, target) pair d = a . b and S = |a| . |b|.  rho / eta are half an ulp of the storage type (relative) and half its
smallest subnormal (conv_reference.RHO / ETA): one rounding of an fp32 value v to storage is off by at most rho |v| + eta.
U = 2^-23.

Rounding model and the bounds that follow from it.
  * Dot products.  Products of two f16 / bf16 values are exact in fp32, and so are the fused products of an fmaf chain;
    the C - 1 additions of a recursive or blocked fp32 sum (tensor cores: blocks of 16 with alignment truncation, see
    conv_reference.py) stay below (C + 20) U S.  The 20 spare terms take the fp32 product with the scale as well.
  * Volume, level 0 (every volume kernel): ref = s d;
        bound = rho |ref| + (1 + rho) |s| (C + 20) U S + eta.
  * Pooled levels rounded once (the tiled kernel: fp32 sums of the fp32 accumulators, one product with s 4^-l, one
    rounding): ref_l = the mean of ref_0 over 2^l x 2^l blocks (floor-halved sizes drop the last row / column).  The 4^l - 1
    additions of the tree are 2l levels deep, each off by at most 2^-24 of its partial sums: l U pool_l(S) on top of the
    accumulators' own error, and the scale product adds 2^-24; so with 3l spare terms
        bound_l = rho |ref_l| + (1 + rho) |s| (C + 20 + 3l) U pool_l(S) + eta.
  * Pooled levels re-rounded at every level (the dense wgmma kernel; the SIMT volume followed by avg_pool2x2): a stored
    value v_l = rt(0.25 (v_0 + v_1 + v_2 + v_3)) of four stored values of level l - 1, each within bound_{l-1} of its
    reference.  The three fp32 additions are off by at most 3 * 2^-24 sum |v_i| (the product with 0.25 is exact), that is
    1.5 U pool(|v|) <= 2 U (pool(|ref_{l-1}|) + pool(bound_{l-1})), then one rounding to storage:
        bound_l = rho |ref_l| + (1 + rho) (pool(bound_{l-1}) + 2 U (pool(|ref_{l-1}|) + pool(bound_{l-1}))) + eta.
  * avg_pool2x2 of stored inputs x: ref = the mean of four; the same sum and rounding:
        bound = rho |ref| + (1 + rho) 2 U pool(|x|) + eta.
  * Lookup from a stored level V (what the kernel stored, read back): the coordinates are float32; as in the kernels,
    x = c 2^-l (exact), a zero window unless |x| < 1e7 and |y| < 1e7, fx = x - floor(x) (exact in fp32), and the tap
    weights w = (1 - fx)(1 - fy), fx (1 - fy), (1 - fx) fy, fx fy.  ref = sum_i w_i V_i over the four taps, in float64 with
    the weights taken from the float32 fx, fy.  The kernels' fp32 weights are off by at most 2 * 2^-24 relative (one
    subtraction, one product), the four products and three additions by 3 * 2^-24 of sum |w_i V_i|: 2.5 U < 4 U, so
        bound = rho |ref| + (1 + rho) 4 U sum |w_i| |V_i| + eta.
    The bound does not depend on the volume's own error, so a wrong tap, weight or channel order (x-major: channel
    l K^2 + i K + j samples x offset i - r, y offset j - r; corr.py:43-47) shows up as many times the bound.
  * On-the-fly, SIMT (corr.cu: corr_onthefly_kernel): the raw dots d_i stay fp32 (within (C + 20) U S_i), then the blend
    with weights w_i s (one more rounding for the scale product: still 4 U):
        bound = rho |ref| + (1 + rho) |s| sum |w_i| ((C + 20) U S_i + 4 U |d_i|) + eta.
  * On-the-fly, tensor cores (corr_onthefly_umma.cu): the scaled dot s d_i is rounded to storage in the accumulator dump
    before the blend, which adds rho |s d_i| + eta per tap (inner_i below), and the blend reads the rounded values:
        inner_i = |s| (rho |d_i| + (1 + rho) (C + 20) U S_i) + eta
        bound   = rho |ref| + (1 + rho) sum |w_i| (inner_i + 4 U (|s| |d_i| + inner_i)) + eta.
The constants follow from the model above; none of them was fitted to measured errors.

``otf_plan`` restates the tensor-core on-the-fly kernel's region rule (the ``geometry`` and ``publish`` lambdas of
corr_onthefly_umma.cu): which queries its region cannot serve (they are flagged and recomputed by the SIMT pass) and how
many 8-row bands each (tile, level) work item multiplies.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch

from conv_reference import ETA, RHO, SENTINEL, U, assert_untouched, assert_within, bits, q, ratio  # noqa: F401

Tensor = torch.Tensor
C_SPARE = 20

# tensor-core on-the-fly kernel geometry (corr_onthefly_umma.cu)
OTF_TILE_H, OTF_TILE_W = 8, 16  # queries per work item
OTF_RW = 32                     # region width (targets)
OTF_MAX_BANDS = 8               # bands of 8 rows at stride 7


# ---------------------------------------------------------------------------------------------------------------------
# volume and pyramid
# ---------------------------------------------------------------------------------------------------------------------
def volume(f1: Tensor, f2: Tensor, scale: float) -> Tuple[Tensor, Tensor]:
    """f1 [B,H1,W1,C], f2 [B,H2,W2,C] (float64 of the stored features) -> (ref, S), each [B*H1*W1, H2, W2]: ref = s d."""
    B, H1, W1, C = f1.shape
    H2, W2 = f2.shape[1:3]
    a = f1.double().reshape(B, H1 * W1, C)
    b = f2.double().reshape(B, H2 * W2, C).transpose(1, 2)
    d = torch.bmm(a, b).reshape(B * H1 * W1, H2, W2)
    S = torch.bmm(a.abs(), b.abs()).reshape(B * H1 * W1, H2, W2)
    return scale * d, S


def pool(x: Tensor, l: int) -> Tensor:
    """Mean over 2^l x 2^l blocks of the last two axes; floor-halved sizes drop the last rows / columns."""
    if l == 0:
        return x
    k = 1 << l
    h, w = x.shape[-2] >> l, x.shape[-1] >> l
    return x[..., :h * k, :w * k].reshape(*x.shape[:-2], h, k, w, k).mean(dim=(-3, -1))


def volume_bound(ref: Tensor, S: Tensor, C: int, scale: float, dtype: torch.dtype) -> Tensor:
    return RHO[dtype] * ref.abs() + (1.0 + RHO[dtype]) * abs(scale) * (C + C_SPARE) * U * S + ETA[dtype]


def pyramid_once(ref0: Tensor, S: Tensor, C: int, scale: float, dtype: torch.dtype, levels: int) -> List[Tuple[Tensor, Tensor]]:
    """[(ref_l, bound_l)] for pooled levels rounded once (the tiled volume kernel)."""
    rho, eta = RHO[dtype], ETA[dtype]
    out = []
    for l in range(levels):
        r = pool(ref0, l)
        out.append((r, rho * r.abs() + (1.0 + rho) * abs(scale) * (C + C_SPARE + 3 * l) * U * pool(S, l) + eta))
    return out


def pool_rerounded(ref_prev: Tensor, bound_prev: Tensor, dtype: torch.dtype) -> Tuple[Tensor, Tensor]:
    """One re-rounded 2x2 pooling step: (ref_l, bound_l) from level l - 1's reference and bound."""
    r = pool(ref_prev, 1)
    pb = pool(bound_prev, 1)
    e = pb + 2.0 * U * (pool(ref_prev.abs(), 1) + pb)
    return r, RHO[dtype] * r.abs() + (1.0 + RHO[dtype]) * e + ETA[dtype]


def pyramid_rerounded(ref0: Tensor, S: Tensor, C: int, scale: float, dtype: torch.dtype, levels: int) -> List[Tuple[Tensor, Tensor]]:
    """[(ref_l, bound_l)] for pooled levels re-rounded at every level (dense wgmma kernel; SIMT volume + avg_pool2x2)."""
    out = [(ref0, volume_bound(ref0, S, C, scale, dtype))]
    for _ in range(1, levels):
        out.append(pool_rerounded(*out[-1], dtype))
    return out


def avg_pool2x2(x: Tensor, dtype: torch.dtype) -> Tuple[Tensor, Tensor]:
    """x [N,H,W,C] (float64 of the stored input) -> (ref, bound) [N,H//2,W//2,C]."""
    xt = x.double().movedim(-1, 1)  # [N,C,H,W]: pool over the last two axes
    ref = pool(xt, 1).movedim(1, -1)
    mag = pool(xt.abs(), 1).movedim(1, -1)
    return ref, RHO[dtype] * ref.abs() + (1.0 + RHO[dtype]) * 2.0 * U * mag + ETA[dtype]


# ---------------------------------------------------------------------------------------------------------------------
# the tiled (T84) layout: element (y, x) of a level's map at ((y >> 2) * tiles_x + (x >> 3)) * 32 + (y & 3) * 8 + (x & 7)
# ---------------------------------------------------------------------------------------------------------------------
def t84_shape(h: int, w: int) -> Tuple[int, int]:
    """(tiles_y, tiles_x) of an h x w map."""
    return (h + 3) // 4, (w + 7) // 8


def t84_offsets(h: int, w: int, device=None) -> Tensor:
    """[h, w] element offsets of the map's in-map elements inside its tiled row of tiles_y * tiles_x * 32 elements."""
    _, tx = t84_shape(h, w)
    y = torch.arange(h, device=device).view(h, 1)
    x = torch.arange(w, device=device).view(1, w)
    return ((y >> 2) * tx + (x >> 3)) * 32 + (y & 3) * 8 + (x & 7)


def t84_read(level: Tensor, h: int, w: int) -> Tensor:
    """Tiled level [Q, tiles_y * tiles_x * 32] -> dense [Q, h, w] (same dtype)."""
    off = t84_offsets(h, w, level.device).reshape(-1)
    return level[:, off].reshape(level.shape[0], h, w)


def t84_write(dense: Tensor, pad_value: float = 0.0) -> Tensor:
    """Dense [Q, h, w] -> tiled [Q, tiles_y * tiles_x * 32]; pad rows / columns hold pad_value."""
    Q, h, w = dense.shape
    ty, tx = t84_shape(h, w)
    out = torch.full((Q, ty * tx * 32), pad_value, dtype=dense.dtype, device=dense.device)
    out[:, t84_offsets(h, w, dense.device).reshape(-1)] = dense.reshape(Q, h * w)
    return out


def t84_pad_mask(h: int, w: int, device=None) -> Tensor:
    """[tiles_y * tiles_x * 32] bool: True at pad elements (rows >= h or columns >= w inside the last tiles)."""
    ty, tx = t84_shape(h, w)
    m = torch.ones(ty * tx * 32, dtype=torch.bool, device=device)
    m[t84_offsets(h, w, device).reshape(-1)] = False
    return m


# ---------------------------------------------------------------------------------------------------------------------
# lookup
# ---------------------------------------------------------------------------------------------------------------------
def window_origin(coords: Tensor, l: int, radius: int) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """coords float32 [Q, 2] -> (x0, y0) int64 window origins (first tap) and (fx, fy) float64 fractions at level l, with
    the kernels' float32 arithmetic: a non-finite (|x| >= 1e7, NaN, inf) coordinate gives the origin -1e6 - r (no tap in
    any map) and zero fractions."""
    c = coords.float() * (2.0 ** -l)
    x, y = c[:, 0], c[:, 1]
    fin = (x.abs() < 1e7) & (y.abs() < 1e7)
    far = torch.full_like(x, -1e6)
    xf = torch.where(fin, torch.floor(x), far)
    yf = torch.where(fin, torch.floor(y), far)
    zero = torch.zeros_like(x)
    fx = torch.where(fin, x - xf, zero)
    fy = torch.where(fin, y - yf, zero)
    return xf.long() - radius, yf.long() - radius, fx.double(), fy.double()


def tap_weights(fx: Tensor, fy: Tensor) -> Sequence[Tuple[int, int, Tensor]]:
    """(dx, dy, weight) of the four bilinear taps."""
    return ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy))


def gather_window(V: Tensor, x0: Tensor, y0: Tensor, K: int, dx: int, dy: int) -> Tensor:
    """V [Q, h, w]; the tap (dx, dy) of every window position -> [Q, K * K] in x-major channel order (i * K + j: x offset i,
    y offset j), zero outside the map."""
    Q, h, w = V.shape
    k = torch.arange(K, device=V.device)
    xi = (x0.to(V.device).view(Q, 1, 1) + k.view(1, K, 1) + dx).expand(Q, K, K)
    yi = (y0.to(V.device).view(Q, 1, 1) + k.view(1, 1, K) + dy).expand(Q, K, K)
    ok = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
    idx = (yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).reshape(Q, K * K)
    v = torch.gather(V.reshape(Q, h * w), 1, idx)
    return torch.where(ok.reshape(Q, K * K), v, torch.zeros_like(v))


def lookup(levels: Sequence[Tensor], coords: Tensor, radius: int, dtype: torch.dtype) -> Tuple[Tensor, Tensor]:
    """levels: float64 [Q, h_l, w_l] of the stored values; coords float32 [Q, 2]; dtype: the output's storage type.
    -> (ref, bound) [Q, L * (2r+1)^2] (pixel-major channel order)."""
    K = 2 * radius + 1
    refs, mags = [], []
    for l, V in enumerate(levels):
        V = V.double()
        x0, y0, fx, fy = window_origin(coords, l, radius)
        fx, fy = fx.to(V.device), fy.to(V.device)
        ref = torch.zeros(V.shape[0], K * K, dtype=torch.float64, device=V.device)
        mag = torch.zeros_like(ref)
        for dx, dy, wt in tap_weights(fx, fy):
            v = gather_window(V, x0, y0, K, dx, dy)
            ref = ref + wt.view(-1, 1) * v
            mag = mag + wt.abs().view(-1, 1) * v.abs()
        refs.append(ref)
        mags.append(mag)
    ref, mag = torch.cat(refs, 1), torch.cat(mags, 1)
    return ref, RHO[dtype] * ref.abs() + (1.0 + RHO[dtype]) * 4.0 * U * mag + ETA[dtype]


def onthefly(f1: Tensor, f2_levels: Sequence[Tensor], coords: Tensor, radius: int, scale: float, dtype: torch.dtype,
             tensor_cores: bool) -> Tuple[Tensor, Tensor]:
    """f1 [B,H,W,C], f2_levels [B,h_l,w_l,C] (float64 of the stored features), coords float32 [B*H*W, 2] ->
    (ref, bound) [B*H*W, L * (2r+1)^2]; ``tensor_cores``: the dump-rounded bound, else the SIMT one."""
    rho, eta = RHO[dtype], ETA[dtype]
    C = f1.shape[-1]
    K = 2 * radius + 1
    s = abs(scale)
    refs, bounds = [], []
    for l, f2 in enumerate(f2_levels):
        d, S = volume(f1, f2, 1.0)
        x0, y0, fx, fy = window_origin(coords, l, radius)
        fx, fy = fx.to(d.device), fy.to(d.device)
        ref = torch.zeros(d.shape[0], K * K, dtype=torch.float64, device=d.device)
        err = torch.zeros_like(ref)
        for dx, dy, wt in tap_weights(fx, fy):
            di = gather_window(d, x0, y0, K, dx, dy)
            Si = gather_window(S, x0, y0, K, dx, dy)
            wa = wt.abs().view(-1, 1)
            ref = ref + scale * wt.view(-1, 1) * di
            acc = (C + C_SPARE) * U * Si
            if tensor_cores:
                inner = s * (rho * di.abs() + (1.0 + rho) * acc) + eta
                err = err + wa * (inner + 4.0 * U * (s * di.abs() + inner))
            else:
                err = err + wa * s * (acc + 4.0 * U * di.abs())
        refs.append(ref)
        bounds.append(rho * ref.abs() + (1.0 + rho) * err + eta)
        del d, S
    return torch.cat(refs, 1), torch.cat(bounds, 1)


# ---------------------------------------------------------------------------------------------------------------------
# the tensor-core on-the-fly kernel's region rule
# ---------------------------------------------------------------------------------------------------------------------
def otf_plan(coords: Tensor, H: int, W: int, levels: int, radius: int = 4) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """coords float32 [B, H, W, 2] -> (nb, bx, by, flags).

    nb, bx, by: int64 [n_items] per work item (item = tile * levels + level, tile = (b * tiles_y + ty) * tiles_x + tx): the
    number of 8-row bands and the region's anchor.  A query of the 8 x 16 tile is live when it is inside the grid, its
    coordinates are finite at that level and its (2r+2)^2 window overlaps the level's map.  The anchor is the smallest
    window origin (x0, y0) over the live queries; By the largest y0; nb = clamp((By + 2r + 1 - by + 6) // 7, 1, 8).  A tile
    without live queries has nb = 0 (no band is loaded) and anchor (0, 0).
    flags: bool [B, H, W], the queries the region cannot serve at some level: live and (cxo + 2r + 2 > 32 or
    ryo + 2r + 1 > 7 nb), (cxo, ryo) = window origin - anchor."""
    B = coords.shape[0]
    D = 2 * radius + 2
    ty_n, tx_n = (H + OTF_TILE_H - 1) // OTF_TILE_H, (W + OTF_TILE_W - 1) // OTF_TILE_W
    Hp, Wp = ty_n * OTF_TILE_H, tx_n * OTF_TILE_W
    c = torch.full((B, Hp, Wp, 2), float("nan"), dtype=torch.float32, device=coords.device)
    c[:, :H, :W] = coords.float()
    inside = torch.zeros((B, Hp, Wp), dtype=torch.bool, device=coords.device)
    inside[:, :H, :W] = True
    BIG = 1 << 40
    nbs, bxs, bys = [], [], []
    flags = torch.zeros((B, H, W), dtype=torch.bool, device=coords.device)
    for l in range(levels):
        hl, wl = H >> l, W >> l
        x0, y0, _, _ = window_origin(c.reshape(-1, 2), l, radius)
        x0, y0 = x0.view(B, Hp, Wp), y0.view(B, Hp, Wp)
        live = inside & (x0 + D - 1 >= 0) & (x0 < wl) & (y0 + D - 1 >= 0) & (y0 < hl)

        def tiles(t):  # [B, Hp, Wp] -> [B, ty, tx, 8 * 16]
            return t.view(B, ty_n, OTF_TILE_H, tx_n, OTF_TILE_W).permute(0, 1, 3, 2, 4).reshape(B, ty_n, tx_n, -1)

        lt, xt, yt = tiles(live), tiles(x0), tiles(y0)
        big = torch.full_like(xt, BIG)
        bx = torch.where(lt, xt, big).amin(-1)
        by = torch.where(lt, yt, big).amin(-1)
        By = torch.where(lt, yt, -big).amax(-1)
        any_live = lt.any(-1)
        nb = torch.div(By + D - 1 - by + 6, 7, rounding_mode="floor").clamp(1, OTF_MAX_BANDS)
        nb = torch.where(any_live, nb, torch.zeros_like(nb))
        bx = torch.where(any_live, bx, torch.zeros_like(bx))
        by = torch.where(any_live, by, torch.zeros_like(by))
        out = lt & (((xt - bx[..., None]) + D > OTF_RW) | ((yt - by[..., None]) + D - 1 > 7 * nb[..., None]))
        flags |= out.view(B, ty_n, tx_n, OTF_TILE_H, OTF_TILE_W).permute(0, 1, 3, 2, 4).reshape(B, Hp, Wp)[:, :H, :W]
        nbs.append(nb.reshape(-1))
        bxs.append(bx.reshape(-1))
        bys.append(by.reshape(-1))
    stack = lambda ts: torch.stack(ts, 1).reshape(-1)  # noqa: E731  (tile-major, level-minor: the kernel's item order)
    return stack(nbs), stack(bxs), stack(bys), flags
