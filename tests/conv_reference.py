"""Float64 reference of the convolution building block (pfb_conv2d) and an error bound per output element (TEST
INFRASTRUCTURE, like gma_oracle.py).  The conformance tests (test_gpu_conv_conformance.py) compare the wgmma and the SIMT
kernels with it; test_conv_reference.py shows on the CPU that the bound rejects plausible kernel bugs.

Reference.  F.conv2d ("same" zero padding, stride 1) in float64 over the inputs, weights and aux operands (h, z, residual,
addend, flow) as they are stored, i.e. already rounded to the storage type; the epilogue is then applied in float64.  On a
GPU the float64 convolutions run on the device.

Bound.  For every output element

    |got - ref| <= rho_out * |ref| + (1 + rho_out) * (L_epi * E_acc + eps_fn) + eta_out,      E_acc = c_acc * 2^-23 * S

  * S = conv(|x|, |w|) + |bias| (or + |addend|) in float64: the sum of the magnitudes of everything the accumulator adds.
  * E_acc bounds the fp32 accumulation error.  The products of two f16 / bf16 values are exact in fp32 (at most 22
    significant bits), and so are the fused products of the fp32 SIMT kernel's fmaf.  What remains are the additions: a
    recursive fp32 sum of n terms is off by at most (n - 1) * u * S (first order), u = 2^-24 for round-to-nearest (the SIMT
    fmaf chain) and 2^-23 when every addition may truncate.  The tensor cores add a block of 16 products to the accumulator
    per K step with alignment truncation (Fasi, Higham, Mikaitis, Pranesh, "Numerical behavior of NVIDIA tensor cores",
    PeerJ CS 2021); that blocked sum stays below (n / 16 + 18) * 2^-23 * S.  With n = KH * KW * Cin + 1 (the bias), both
    kernels are covered by c_acc = n + 20: the 20 spare terms also take the epilogue's own fp32 roundings of quantities
    bounded by S (the bias or addend add, the scale product, the residual add).
  * rho_out is half an ulp of the output type relative to the value (2^-11 f16, 2^-8 bf16, 2^-24 fp32) and eta_out half
    the smallest subnormal (2^-25 f16, 2^-134 bf16, 2^-150 fp32): the one rounding of the fp32 result to storage.  The
    factor (1 + rho_out) is there because the value that is rounded is the fp32 result, not ref.
  * L_epi is the epilogue's Lipschitz factor in the accumulator: |scale| (LINEAR, LINEAR_F32, AXPY), 1 (RELU, the
    APPEND_FLOW channels), max |gelu'| = Phi(sqrt 2) + sqrt 2 * phi(sqrt 2) < 1.13 (GELU, RESIDUAL_GELU; times
    1.13 * |1 + post_w| for the second step), 1/4 (sigmoid: z), |h| / 4 (r * h), |z| (tanh' <= 1: GRU_Q).
  * eps_fn bounds the fp32 arithmetic of the epilogue function itself, with |v| <= S for its argument v:
      - sigmoid 1 / (1 + __expf(-v)) with __fdividef: __expf is within (2 + 1.2 |v|) ulp (CUDA C++ Programming Guide,
        intrinsic functions), the add 1/2 ulp, __fdividef 2 ulp; through sigma * (1 - sigma) <= 1/4 this is at most
        2^-23 * (3 + 0.3 |v|).  The SIMT kernel's expf / IEEE division is more accurate.
      - tanh as 1 - 2 / (1 + __expf(2v)): with d(2 / (1 + e)) / (e / e) <= 1/2 the quotient is within
        2^-23 * (1 + 1.2 |v|) + 2 * 1.25 * 2^-22 and the final subtraction adds 2^-24: 2^-23 * (7 + 1.2 |v|).
      - gelu 0.5 x (1 + erff(x / sqrt 2)): erff is within 2 ulp, i.e. 2^-23 for values <= 1; with the argument product,
        the add and the two products at most 2.25 * 2^-23 * |x| <= 2^-21 * |x|.
      - the gate and axpy combinations (1 - z) h + z q, r * h and h + s * v: three fp32 roundings of terms bounded by
        |h| + 1 (or |h| + |s| S): 2^-22 of that.
    The constants follow from the model above; none of them was fitted to measured errors.

Every output buffer is filled with a sentinel first; ``assert_untouched`` then checks that no column outside the layer's
output range (and so no pad column of Cout_pad_k) changed.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

# pfb_epilogue (include/ptlflow_b200.h)
LINEAR, RELU, GRU_ZR, GRU_Q, FLOW, RELU_APPEND_FLOW, AXPY, LINEAR_F32, GELU, RESIDUAL_GELU, LINEAR_APPEND_FLOW = range(11)
EPI_NAMES = {LINEAR: "linear", RELU: "relu", GRU_ZR: "gru_zr", GRU_Q: "gru_q", RELU_APPEND_FLOW: "relu_append_flow", AXPY: "axpy",
             LINEAR_F32: "linear_f32", GELU: "gelu", RESIDUAL_GELU: "residual_gelu", LINEAR_APPEND_FLOW: "linear_append_flow"}

RHO = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -24}
ETA = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -134, torch.float32: 2.0 ** -150}
U = 2.0 ** -23
C_SPARE = 20
GELU_LIP = 1.13
SENTINEL = -4321.0


def q(t: Tensor, dtype: torch.dtype) -> Tensor:
    """t rounded to the storage type, as float64."""
    return t.to(dtype).double()


def conv_terms(xs: Sequence[Tensor], weight: Tensor, bias: Optional[Tensor] = None, addend: Optional[Tensor] = None,
               per_sample: bool = False, stride: int = 1) -> Tuple[Tensor, Tensor, int]:
    """Pre-activation and magnitude sum of a convolution, float64, pixel-major.

    xs: the sources [B,H,W,Ci] (float64, storage-rounded), concatenated along channels.  weight: [Cout, sum Ci, KH, KW], or
    with ``per_sample`` [B, Cout, sum Ci] (1x1, one matrix per sample).  bias [Cout] or addend [B,H,W,Cout] (instead of the
    bias).  ``stride``: of the convolution, with the same zero padding KH // 2, KW // 2 (the encoders' 7x7 stride-2 conv1).
    Returns (acc, S, n): acc = conv + bias / addend and S = conv(|x|, |w|) + |bias| / |addend|, both [B,Ho,Wo,Cout], and n,
    the number of terms each output adds."""
    x = torch.cat([t.double() for t in xs], -1)
    w = weight.double()
    if per_sample:
        acc = torch.einsum("bhwc,boc->bhwo", x, w)
        S = torch.einsum("bhwc,boc->bhwo", x.abs(), w.abs())
        n = w.shape[2]
    else:
        kh, kw = w.shape[2], w.shape[3]
        xn = x.permute(0, 3, 1, 2)
        acc = F.conv2d(xn, w, padding=(kh // 2, kw // 2), stride=stride).permute(0, 2, 3, 1)
        S = F.conv2d(xn.abs(), w.abs(), padding=(kh // 2, kw // 2), stride=stride).permute(0, 2, 3, 1)
        n = kh * kw * w.shape[1]
    if addend is not None:
        acc, S = acc + addend.double(), S + addend.double().abs()
    elif bias is not None:
        acc, S = acc + bias.double(), S + bias.double().abs()
    return acc.contiguous(), S.contiguous(), n + 1


def gelu64(x: Tensor) -> Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def epilogue(epi: int, acc: Tensor, S: Tensor, n: int, dtype: torch.dtype, *, scale: float = 1.0, h: Optional[Tensor] = None,
             z: Optional[Tensor] = None, hidden: int = 0, residual: Optional[Tensor] = None, post_w: Optional[Tensor] = None,
             post_b: Optional[Tensor] = None, flow: Optional[Tensor] = None) -> Dict[str, Tuple[Tensor, Tensor]]:
    """The epilogue in float64 and its bound: {"out": (ref, bound)} (+ "z" for GRU_ZR), each [B,H,W,C].  ``dtype`` is the
    output's storage type (fp32 for LINEAR_F32).  h / z: [B,H,W,hidden] (GRU; AXPY reads h as its residual), residual
    [B,H,W,Cout] (the operand's channels already selected), post_w / post_b [Cout], flow [B,H,W,2]; all float64 of the stored
    values."""
    rho, eta = RHO[dtype], ETA[dtype]
    E = (n + C_SPARE) * U * S

    def pair(ref, err):
        return ref, rho * ref.abs() + (1.0 + rho) * err + eta

    if epi in (LINEAR, LINEAR_F32):
        return {"out": pair(scale * acc, abs(scale) * E)}
    if epi == RELU:
        return {"out": pair(acc.clamp_min(0.0), E)}
    if epi in (RELU_APPEND_FLOW, LINEAR_APPEND_FLOW):
        v = acc.clamp_min(0.0) if epi == RELU_APPEND_FLOW else acc
        f = flow.double()
        return {"out": pair(torch.cat([v, f], -1), torch.cat([E, torch.zeros_like(f)], -1))}
    if epi == AXPY:
        hh = h.double()[..., :acc.shape[-1]]
        return {"out": pair(hh + scale * acc, abs(scale) * E + 2.0 ** -22 * (hh.abs() + abs(scale) * S))}
    if epi == GELU:
        return {"out": pair(gelu64(acc), GELU_LIP * E + 2.0 ** -21 * S)}
    if epi == RESIDUAL_GELU:
        r = residual.double()
        u = r + acc
        Su = r.abs() + S
        y = gelu64(u)
        ey = GELU_LIP * E + 2.0 ** -21 * Su
        if post_w is None:
            return {"out": pair(y, ey)}
        g = 1.0 + post_w.double()
        u2 = y * g + post_b.double()
        S2 = y.abs() * g.abs() + post_b.double().abs()
        return {"out": pair(gelu64(u2), GELU_LIP * (g.abs() * ey + 2.0 ** -22 * S2) + 2.0 ** -21 * S2)}
    if epi == GRU_ZR:
        sig = torch.sigmoid(acc)
        es = 0.25 * E + U * (3.0 + 0.3 * S)
        hh = h.double()
        zr = sig[..., :hidden]
        rh = sig[..., hidden:] * hh
        return {"z": pair(zr, es[..., :hidden]),
                "out": pair(rh, hh.abs() * es[..., hidden:] + 2.0 ** -22 * (hh.abs() + 1.0))}
    if epi == GRU_Q:
        hh, zz = h.double(), z.double()
        th = torch.tanh(acc)
        et = E + U * (7.0 + 1.2 * S)
        return {"out": pair((1.0 - zz) * hh + zz * th, zz.abs() * et + 2.0 ** -22 * (hh.abs() + 1.0))}
    raise ValueError(f"epilogue {epi} has no reference here")


def ratio(got: Tensor, ref: Tensor, bound: Tensor) -> Tensor:
    """|got - ref| / bound per element (inf where got is not finite)."""
    g = got.double().to(ref.device)
    r = (g - ref).abs() / bound
    return torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))


def max_ratio(got: Tensor, ref: Tensor, bound: Tensor) -> float:
    return ratio(got, ref, bound).max().item()


def within(got: Tensor, ref: Tensor, bound: Tensor) -> bool:
    return max_ratio(got, ref, bound) <= 1.0


def assert_within(got: Tensor, ref: Tensor, bound: Tensor, what: str = "") -> float:
    """Asserts every element is inside its bound; returns max(err / bound)."""
    r = ratio(got, ref, bound)
    worst = r.max().item()
    if not worst <= 1.0:
        bad = (~(r <= 1.0)).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} of {r.numel()} elements outside the bound, max err/bound {worst:.3g}; "
                             f"first at {i}: got {got[i].item()!r}, ref {ref[i].item()!r}, bound {bound[i].item():.3g}")
    return worst


def bits(t: Tensor) -> Tensor:
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def assert_untouched(buf: Tensor, before: Tensor, lo: int, hi: int, what: str = "") -> None:
    """Every column of buf [..., C] outside [lo, hi) holds exactly what it held before (bitwise)."""
    for a, b in ((buf[..., :lo], before[..., :lo]), (buf[..., hi:], before[..., hi:])):
        if a.numel() and not torch.equal(bits(a), bits(b)):
            raise AssertionError(f"{what}: columns outside [{lo}, {hi}) were written")
