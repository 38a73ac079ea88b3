"""Float64 references of the kernels that carry the fp32 flow, with an error bound per output element (TEST INFRASTRUCTURE,
like conv_reference.py): the flow head's coordinate update, the convex upsamplers (8x, 4x, 2x and CCMR's handover) and the
bilinear resamplers upflow8 / upflow2 / downflow.  test_gpu_flow_conformance.py compares the kernels with them element by
element; test_flow_reference.py shows on the CPU that the bounds admit correct fp32 implementations and reject plausible
bugs.  u = 2^-24 is the unit roundoff of fp32 (round to nearest).  None of the constants below was fitted to measured errors.

Flow head (3x3 conv, Cin -> 2, fused with coords += delta; flow = coords - (x, y)).  conv_reference.epilogue(FLOW) holds it:
E_acc of conv_reference with n = 9 Cin + 1 plus the roundings of the coordinate add and of the grid subtraction.  The three
kernels that compute it:
  * conv_cout2_flow_kernel (f16 / bf16): per-lane fmaf chains, a shuffle tree, then (c + acc) + bias.  Every addition is one
    rounding of a partial sum bounded by S: at most (9 Cin + 1 - 1) u S in all, inside E_acc = (n + C_SPARE) 2^-23 S.
  * the SIMT FLOW epilogue: one fmaf chain along K, + bias, + c.
  * the tensor-core route: a LINEAR_F32 1x1 GEMM of the 18 per-tap weight rows (engine._taps: row tap * 2 + o) writes T[p][tap *
    2 + o] = sum_c x[p][c] w[o][c][tap], each within (Cin / 16 + 18) 2^-23 S_tap (the blocked tensor-core sum, see
    conv_reference), S_tap its magnitude sum; flow_tap_gather_kernel then adds the bias and the 9 in-image taps in fp32, 9
    roundings of sums bounded by S = |bias| + sum_tap S_tap: 4.5 * 2^-23 S.  Together (Cin / 16 + 22.5) 2^-23 S, which is below
    (9 Cin + 1 + C_SPARE) 2^-23 S for every Cin >= 1: the same E_acc covers it.

Convex upsample by F (F in {2, 4, 8}; misc.cu convex_upsample_kernel, msraft.cu convex_upsample2x_kernel).  Output (sy, sx) of
the coarse pixel p is sum_t softmax_t(m) a_t over the 9 taps t = 3 (dy + 1) + (dx + 1) of mask channel t F^2 + sy F + sx,
a_t = F * fp32(c_t - g_t) for an in-image neighbour (g_t its grid position, 0 in mode 1) and 0 outside the image; the
out-of-image taps stay in the softmax's denominator (the zero-padded unfold).  Mode 2 adds the fine grid (F x + sx, F y + sy).
With x_t = m_t - max m (<= 0), w_t the exact softmax weights and s their sum, the kernel computes
  * e_t = expf(fl(m_t - max)): the subtraction is off by u |x_t| relative, expf by at most 2 ulp <= 4 u (CUDA C++ Programming
    Guide, single-precision mathematical functions, full range), and a subnormal result by at most 2^-148 absolute;
  * ax = fmaf(e_t, a_t, ax) over the in-image taps: term t passes through at most 9 roundings; sum += e_t: 8 roundings;
  * ax * (1 / sum): two more roundings of the result.
To first order the numerator's relative error per term is (4 + 9 + |x_t|) u and the denominator's (4 + 8) u + u sum_t w_t |x_t|
(a weighted mean), so with Sa = sum_t w_t |a_t| >= |ref|:
    |got - ref| <= u (C_CONVEX Sa + sum_t w_t |a_t| |x_t| + |ref| sum_t w_t |x_t|) + 2^-140 (sum_t |a_t| + |ref|)
with C_CONVEX = 13 + 12 + 2 = 27, plus 1 for every second-order term: 28.  (sum_t w_t |x_t| <= 9 / e: the |x_t| terms stay
small.)  The same constant admits a softmax that divides each weight first (torch.softmax, the models' reference): its
weights are within (2 + 8 + 1 + |x_t|) u each (exp 1 ulp, sum, division) and the 9 products and 8 additions add 9 more.
Mode 2's fp32 add of the grid is one more rounding: + u |ref + grid|.

Bilinear resamplers (upflow8: 8 * up8(flow); upflow2: 2 * up2(flow); downflow: (su u, sv v) of a resize to (oh, ow)), all
F.interpolate(bilinear, align_corners=True).  The source index of output o (the window's offset pad included) follows ATen's
fp32 arithmetic exactly, computed here in numpy float32: scale = fp32(in - 1) / fp32(out - 1) (0 when out == 1),
src = fp32(scale * (o + pad)), i0 = floor(src), i1 = i0 + (i0 < in - 1), lam = src - i0 (exact).  The blend of the four
neighbours is float64.  Its fp32 evaluation (1 - l)((1 - k) f00 + k f01) + l((1 - k) f10 + k f11) rounds each term at most 6
times (the weight, the inner product and sum, the outer weight, product and sum), upflow8 / upflow2 round the flow c - g once
before, downflow its scale product once after:
    |got - ref| <= C_BLEND u |mult| S,    S = the blend of |f|,    C_BLEND = 8.
A kernel with other index arithmetic (align_corners=False, a float64 scale, another rounding of src) moves lam by far more than
that wherever neighbouring values differ.
"""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np
import torch

Tensor = torch.Tensor

U24 = 2.0 ** -24
C_CONVEX = 28
C_BLEND = 8
ETA_EXP = 2.0 ** -140
SENTINEL = -4321.0


def grid_xy(B: int, H: int, W: int, device=None) -> Tensor:
    """float64 [B,H,W,2]: (x, y) of every pixel."""
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=device), torch.arange(W, dtype=torch.float64, device=device),
                            indexing="ij")
    return torch.stack([xs, ys], -1).expand(B, H, W, 2)


def to_nchw(t: Tensor, F: int) -> Tensor:
    """[B,H,W,F,F,2] (coarse pixel, sy, sx, component) -> [B,2,F H,F W]."""
    B, H, W = t.shape[:3]
    return t.permute(0, 5, 1, 3, 2, 4).reshape(B, 2, F * H, F * W)


def convex(coords: Tensor, mask: Tensor, F: int, mode: int = 0) -> Tuple[Tensor, Tensor]:
    """Reference and bound of the convex F x upsample, float64 [B,2,F H,F W] each (the full grid; the kernels' windows are crops).
    coords fp32 [B,H,W,2]; mask [B,H,W,9 F^2] as stored (channel t F^2 + sy F + sx).  mode 0: the flow; 1: the absolute
    coordinates (g = 0); 2: the flow plus the fine grid."""
    B, H, W, _ = coords.shape
    dev = coords.device
    c32 = coords.float()
    g32 = grid_xy(B, H, W, dev).float() if mode != 1 else torch.zeros_like(c32)
    a = F * (c32 - g32).double()  # the fp32 difference, as every implementation forms it; times F exactly
    ap = torch.nn.functional.pad(a.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)  # zero outside the image
    taps = torch.stack([ap[:, dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], 3)  # [B,H,W,9,2]
    m = mask.double().view(B, H, W, 9, F, F)
    x = m - m.amax(3, keepdim=True)
    e = torch.exp(x)
    w = e / e.sum(3, keepdim=True)  # [B,H,W,9,F,F]
    ta = taps[:, :, :, :, None, None, :]  # [B,H,W,9,1,1,2]
    wt = w[..., None]
    ref = (wt * ta).sum(3)  # [B,H,W,F,F,2]
    Sa = (wt * ta.abs()).sum(3)
    Sx = (wt * ta.abs() * x[..., None].abs()).sum(3)
    Wx = (w * x.abs()).sum(3)[..., None]
    bound = U24 * (C_CONVEX * Sa + Sx + ref.abs() * Wx) + ETA_EXP * (taps.abs().sum(3)[:, :, :, None, None, :] + ref.abs())
    ref, bound = to_nchw(ref, F), to_nchw(bound, F)
    if mode == 2:
        fine = grid_xy(B, F * H, F * W, dev).permute(0, 3, 1, 2)
        ref = ref + fine
        bound = bound + U24 * ref.abs()
    return ref, bound


def onehot_expected(coords: Tensor, tap: Tensor, F: int, mode: int = 0) -> Tensor:
    """What a one-hot mask gives exactly: fp32 [B,2,F H,F W], F * fp32(c_t - g_t) of the dominant tap t = tap[b,y,x,sy,sx] (0
    outside the image); mode 1 without the grid, mode 2 plus the fine grid in fp32."""
    B, H, W, _ = coords.shape
    dev = coords.device
    c32 = coords.float()
    g32 = grid_xy(B, H, W, dev).float() if mode != 1 else torch.zeros_like(c32)
    a = F * (c32 - g32)
    ap = torch.nn.functional.pad(a.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    taps = torch.stack([ap[:, dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], 3)  # [B,H,W,9,2]
    idx = tap.long()[..., None].expand(B, H, W, F, F, 2).reshape(B, H, W, F * F, 2)
    got = torch.gather(taps, 3, idx.clamp(0, 8)).view(B, H, W, F, F, 2)
    out = to_nchw(got, F)
    if mode == 2:
        out = out + grid_xy(B, F * H, F * W, dev).permute(0, 3, 1, 2).float()
    return out


def aten_source_index(n_in: int, n_out: int, o: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """ATen's align_corners=True source index of the output indices ``o`` (of a resize n_in -> n_out), in fp32:
    -> (i0, i1, lam) with lam float32."""
    f32 = np.float32
    scale = f32(n_in - 1) / f32(n_out - 1) if n_out > 1 else f32(0.0)
    src = (scale * np.asarray(o).astype(f32)).astype(f32)
    i0 = np.floor(src).astype(np.int64)
    i1 = i0 + (i0 < n_in - 1).astype(np.int64)
    lam = (src - i0.astype(f32)).astype(f32)
    return i0, i1, lam


def bilinear(f: Tensor, full_hw, out_hw=None, pad=(0, 0), mult: Tuple[float, float] = (1.0, 1.0)) -> Tuple[Tensor, Tensor]:
    """mult[c] * F.interpolate(f, full_hw, bilinear, align_corners=True), the window out_hw at pad: (ref, bound), float64
    [B,2,oh,ow].  f: [B,2,H,W] (float64 of the values the kernel reads, or forms in one fp32 rounding)."""
    B, C, H, W = f.shape
    oh, ow = out_hw or full_hw
    y0, y1, ly = aten_source_index(H, full_hw[0], np.arange(oh) + pad[0])
    x0, x1, lx = aten_source_index(W, full_hw[1], np.arange(ow) + pad[1])
    dev = f.device
    t = lambda a: torch.as_tensor(a, device=dev)  # noqa: E731
    y0, y1, x0, x1 = t(y0), t(y1), t(x0), t(x1)
    ly = t(ly.astype(np.float64))[:, None]
    lx = t(lx.astype(np.float64))[None, :]
    f = f.double()

    def blend(v):
        r0, r1 = v[:, :, y0], v[:, :, y1]
        return (1 - ly) * ((1 - lx) * r0[..., x0] + lx * r0[..., x1]) + ly * ((1 - lx) * r1[..., x0] + lx * r1[..., x1])

    m = torch.tensor(mult, dtype=torch.float64, device=dev).view(1, C, 1, 1)
    ref = m * blend(f)
    bound = C_BLEND * U24 * m.abs() * blend(f.abs())
    return ref, bound


def flow_of(coords: Tensor) -> Tensor:
    """float64 [B,2,H,W] of the flow c - g of fp32 coordinates [B,H,W,2] (exact)."""
    B, H, W, _ = coords.shape
    return (coords.double() - grid_xy(B, H, W, coords.device)).permute(0, 3, 1, 2)


def upflow(coords: Tensor, F: int, out_hw=None, pad=(0, 0)) -> Tuple[Tensor, Tensor]:
    """upflow8 (F = 8, from the coordinates) of the window out_hw at pad."""
    B, H, W, _ = coords.shape
    return bilinear(flow_of(coords), (F * H, F * W), out_hw, pad, (float(F), float(F)))


def upflow2(flow: Tensor, out_hw=None, pad=(0, 0)) -> Tuple[Tensor, Tensor]:
    """upflow2 of the fp32 flow [B,2,H,W]."""
    H, W = flow.shape[-2:]
    return bilinear(flow, (2 * H, 2 * W), out_hw, pad, (2.0, 2.0))


def downflow_scales(H: int, W: int, oh: int, ow: int) -> Tuple[float, float]:
    """(su, sv): the Python floats ow / W and oh / H as the fp32 tensor product rounds them."""
    return float(np.float32(ow / W)), float(np.float32(oh / H))


def downflow(flow: Tensor, out_hw) -> Tuple[Tensor, Tensor]:
    H, W = flow.shape[-2:]
    return bilinear(flow, tuple(out_hw), mult=downflow_scales(H, W, *out_hw))


def ratio(got: Tensor, ref: Tensor, bound: Tensor) -> Tensor:
    """|got - ref| / bound per element (inf where got is not finite; 0 / 0 counts as inside)."""
    g = got.double().to(ref.device)
    d = (g - ref).abs()
    r = torch.where(d == 0, torch.zeros_like(d), d / bound)
    return torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))


def assert_within(got: Tensor, ref: Tensor, bound: Tensor, what: str = "") -> float:
    """Every element inside its bound; returns max(err / bound)."""
    r = ratio(got, ref, bound)
    worst = r.max().item() if r.numel() else 0.0
    if not worst <= 1.0:
        bad = (~(r <= 1.0)).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} of {r.numel()} elements outside the bound, max err/bound {worst:.3g}; "
                             f"first at {i}: got {got[i].item()!r}, ref {ref[i].item()!r}, bound {bound[i].item():.3g}")
    return worst


def max_ratio(got: Tensor, ref: Tensor, bound: Tensor) -> float:
    return ratio(got, ref, bound).max().item()
