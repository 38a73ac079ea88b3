"""Float64 references of the encoders' normalisation passes (csrc/encoder.cu) and of the two first convolutions
(csrc/first_conv.cu), each with an error bound per output element (TEST INFRASTRUCTURE, like conv_reference.py, whose RHO /
ETA store model, accumulator bound and sentinel checks are reused here).  test_gpu_encoder_conformance.py compares the kernels
with it; test_norm_reference.py shows on the CPU that the bounds reject plausible kernel bugs.

Operations, on the values as stored (already rounded to the storage type), in float64:

    instance norm   y = (x - mean) * rstd,  rstd = 1 / sqrt(var + eps),  mean / var over the H x W pixels of one (image, channel)
    group norm      y = (x + b - mean) * rstd * gamma + beta,  mean / var of x + b over the pixels of `group` channels
    bias_act        y = x + b
    then            y -> relu(y) (optional) -> relu(res + y) (optional)

Model of the kernels.  u = 2^-24 is the unit roundoff of fp32 (round to nearest), U64 = 2^-53 that of fp64.

  * Sums.  Per (image, channel) the statistics kernel keeps the sums of x and x^2 in fp32 chains of at most K terms each and
    combines the chains in fp64 (exact conversion, fp64 atomics).  Recursive summation with at most K roundings on any term's
    path gives |s^ - s| <= gamma_K * sum|x| and |q^ - q| <= gamma_K * sum x^2, gamma_K = K u / (1 - K u) (Higham, "Accuracy
    and Stability of Numerical Algorithms", 2nd ed., Lemma 3.1 and section 4.2).  x^2 is exact in fp32 for f16 / bf16 storage
    (at most 22 significant bits) and fmaf(x, x, q) rounds once per term for fp32 storage.  K:
      - launch_stats (pfb_instance_norm_act, pfb_group_norm_act), 256 threads, pixels per block P = 64 / 256 / 768 / 1536 for
        HW < 1024 / < 8192 / < 65536 / larger, C/8 channel octets, L = 256 // (C/8) pixel lanes: each thread adds
        m = ceil(min(P, HW) / L) pixels; when C/8 is a power of two <= 32 the lanes of a warp that share an octet are folded by
        a shuffle tree of d = log2(32 / (C/8)) levels and one lane per warp adds into shared memory (A = 8 warps), otherwise
        every lane adds into shared memory (d = 0, A = L).  A term's path has at most (m - 1) + d + (A - 1) fp32 roundings
        (each chain's first addition is into zero, hence exact); K = m + d + A + 1 leaves one for the rounding of x^2 in
        fp32 storage, one for the fp64 combination of the blocks (at most HW / P additions of relative size 2^-53, far
        below one fp32 rounding) and one spare.  stats_k() computes it: 59 for config 2's layer1 (HW = 112640, C = 64),
        389 at its largest (C = 512, HW >= 65536: four lanes of 384 pixels each).
      - pfb_first_conv7x7s2's epilogue: a thread adds 2 x 32 pixels of one channel per work item into fp32 registers over all
        the work items of its CTA and flushes them in fp64 when the image changes: K = 64 * items per CTA + 1 (first_conv_k).
        Its sums are of v = fl(acc + bias), the fp32 accumulator, not of the stored output; each v is within
        E = (n + 20) 2^-23 S of the exact value (conv_reference), which adds sum E to the error of s and sum E (2|v| + E) to
        that of q.
  * Variance.  mean = s / n and var = max(q / n - mean^2, 0) in fp64.  With dm = ds / n the error of mean,
    |var^ - var| <= dq / n + dm (2 |mean| + dm) + 8 U64 (q / n + mean^2): the one-pass formula amplifies the error of s by
    2 |mean| / n, a term that grows with (mean / sigma)^2 relative to var.  It is kept as it is: this is the accuracy the
    one-pass algorithm has.
  * Group norm.  The sums of the group's channels are combined with the producer's bias folded in fp64:
    s_g = sum_k s_k + b_k HW, q_g = sum_k q_k + 2 b_k s_k + b_k^2 HW, so ds_g = sum ds_k and dq_g = sum dq_k + 2 |b_k| ds_k.
  * rstd = rsqrtf((float) var + eps): the conversion and the add are one fp32 rounding each, rsqrtf is within 2 ulp (2^-22
    relative; CUDA C++ Programming Guide, mathematical functions).  So (float) var + eps lies in [v - D, v + D],
    v = var + eps, D = |var^ - var| + 3 u (var + |var^ - var| + eps), and never below eps (1 - 2u) since var^ >= 0; rstd^ lies
    between (v + D)^-1/2 (1 - 2^-22) and max(v - D, eps (1 - 2u))^-1/2 (1 + 2^-22).  Dr is the larger distance of those ends
    from rstd and R the upper end.  No first-order expansion: the interval stays valid when D is not small against v (a
    constant channel, where var = 0 and v = eps).
  * Scale and shift.  Instance norm: sc = rstd^, sh = fl(fl(-mean^) rstd^), two fp32 roundings of |mean^| R.  Group norm (or
    any bias / affine): sc = fl(rstd^ g) and sh = fl((b - mean^) rstd^ g + beta) in fp64 rounded once to fp32.  The bound
    takes both: u R |g| |x| + 2 u (|b| + |mean| + dm) R |g| + u |beta|.  Then o = fmaf(x, sc, sh) differs from the reference
    y = (x + b - mean) rstd g + beta by at most |g| (|x + b - mean| Dr + dm R) + the roundings above, plus u |o| for the fmaf.
  * bias_act: o = fmaf(x, 1, b), one rounding: u |x + b|.
  * Output.  ReLU is 1-Lipschitz; the residual join relu(res + o) is one more fp32 rounding, u (|res| + |o|); the store to the
    storage type is RHO |ref| + ETA, with the factor (1 + RHO) on the error because the value rounded is the fp32 result.

convf1 (pfb_flow_conv7x7) splits the fp32 flow f into hi = fl_T(f) and lo = fl_T(f - hi) (f - hi is exact in fp32) and
multiplies both halves with the storage-type weights on the tensor cores.  f - hi - lo is the rounding error of lo:
|f - hi - lo| <= u_T |f - hi| <= u_T^2 |f|, u_T = 2^-11 (f16) or 2^-8 (bf16), so rho_split = 2^-22 in f16 and 2^-16 in bf16,
plus, in f16, half the smallest subnormal (2^-25) where lo (or hi) is subnormal.  Its bound is conv_reference's bound of the
7x7 convolution of the two halves (4 input channels, n = 197 with the bias) plus conv(rho_split |f| + eta_split, |w|).  The
header's "no precision lost against the fp32 SIMT kernel" holds in f16 (hi + lo carry 22 bits, the products stay exact) and
not in bf16 (16 bits: the lo half's own rounding, 2^-16 relative, is larger than fp32's 2^-24).

None of the constants above was fitted to measured errors.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

import conv_reference as R

Tensor = torch.Tensor

U32 = 2.0 ** -24
U64 = 2.0 ** -53
RSQRT_REL = 2.0 ** -22  # rsqrtf: 2 ulp
SPLIT = {torch.float16: (2.0 ** -22, 2.0 ** -25), torch.bfloat16: (2.0 ** -16, 2.0 ** -134)}  # (rho_split, eta_split)
FC_PIX = 128  # output pixels per first-conv work item (the MMA's N)


def gamma_k(k: int) -> float:
    return k * U32 / (1.0 - k * U32)


def stats_k(HW: int, C: int) -> int:
    """K of launch_stats (csrc/encoder.cu) for an HW-pixel image with C channels: see the module docstring."""
    ppb = 1536 if HW >= 65536 else (768 if HW >= 8192 else (256 if HW >= 1024 else 64))
    c8n = C // 8
    lanes = 256 // c8n
    m = -(-min(ppb, HW) // lanes)
    pow2 = (c8n & (c8n - 1)) == 0 and c8n <= 32 and 256 % c8n == 0
    d = int(math.log2(32 // c8n)) if pow2 else 0
    a = 8 if pow2 else lanes
    return m + d + a + 1


def first_conv_items(N: int, Ho: int, Wo: int, sms: int) -> Tuple[int, int]:
    """(work items, items per CTA) of pfb_first_conv7x7s2 on ``sms`` multiprocessors: an item is 2 output rows x 128 pixels."""
    n_items = N * (-(-Ho // 2)) * (-(-Wo // FC_PIX))
    grid = min(sms, n_items)
    return n_items, -(-n_items // grid)


def first_conv_k(per_cta: int) -> int:
    return 64 * per_cta + 1


def sums(x: Tensor) -> Tuple[Tensor, Tensor]:
    """float64 (sum x, sum x^2) per (image, channel) of x [B,H,W,C]: [B,C] each."""
    x = x.double()
    return x.sum(dim=(1, 2)), (x * x).sum(dim=(1, 2))


def sum_errors(x: Tensor, k: int) -> Tuple[Tensor, Tensor]:
    """Bounds on the errors of the fp32-chained sums of x [B,H,W,C] with chains of at most k terms: [B,C] each."""
    x = x.double()
    g = gamma_k(k)
    return g * x.abs().sum(dim=(1, 2)), g * (x * x).sum(dim=(1, 2))


def conv_sum_errors(acc: Tensor, E: Tensor, k: int) -> Tuple[Tensor, Tensor]:
    """The same for sums of fp32 accumulator values within E of acc (the first convolution's epilogue statistics)."""
    g = gamma_k(k)
    m = acc.abs() + E
    return (g * m.sum(dim=(1, 2)) + E.sum(dim=(1, 2)),
            g * (m * m).sum(dim=(1, 2)) + (E * (2.0 * acc.abs() + E)).sum(dim=(1, 2)))


def _rstd(var: Tensor, dvar: Tensor, eps: float) -> Tuple[Tensor, Tensor, Tensor]:
    """(rstd, Dr, R): 1 / sqrt(var + eps), a bound on |rstd^ - rstd| and an upper bound on rstd^."""
    v = var + eps
    D = dvar + 3.0 * U32 * (var + dvar + eps)
    rstd = v.rsqrt()
    hi = (v - D).clamp_min(eps * (1.0 - 2.0 * U32)).rsqrt() * (1.0 + RSQRT_REL)
    lo = (v + D).rsqrt() * (1.0 - RSQRT_REL)
    return rstd, torch.maximum(hi - rstd, rstd - lo), hi


def _out(y: Tensor, err: Tensor, dtype: torch.dtype, relu: bool, residual: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """The fmaf's rounding, then ReLU, the residual join and the store: (ref, bound)."""
    err = err + U32 * (y.abs() + err)
    if relu:
        y = y.clamp_min(0.0)
    if residual is not None:
        r = residual.double()
        err = err + U32 * (r.abs() + y.abs() + err)
        y = (r + y).clamp_min(0.0)
    rho, eta = R.RHO[dtype], R.ETA[dtype]
    return y, rho * y.abs() + (1.0 + rho) * err + eta


def normalize(x: Tensor, s: Tensor, q: Tensor, ds: Tensor, dq: Tensor, dtype: torch.dtype, *, eps: float = 1e-5,
              relu: bool = False, residual: Optional[Tensor] = None, bias: Optional[Tensor] = None,
              gamma: Optional[Tensor] = None, beta: Optional[Tensor] = None, group: int = 1) -> Tuple[Tensor, Tensor]:
    """Instance norm (group 1, no bias / affine) or group norm of x [B,H,W,C] (float64 of the stored values) from per-(image,
    channel) sums s, q [B,C] of x (without the bias) that are within ds, dq of the exact sums; (ref, bound), [B,H,W,C]."""
    x = x.double()
    B, H, W, C = x.shape
    HW = H * W
    G = C // group
    b = bias.double().to(x.device) if bias is not None else torch.zeros(C, dtype=torch.float64, device=x.device)
    sg = (s + b * HW).view(B, G, group).sum(-1)
    qg = (q + 2.0 * b * s + b * b * HW).view(B, G, group).sum(-1)
    qabs = (q + 2.0 * b.abs() * s.abs() + b * b * HW).view(B, G, group).sum(-1)
    dsg = ds.view(B, G, group).sum(-1)
    dqg = (dq + 2.0 * b.abs() * ds).view(B, G, group).sum(-1)
    n = float(HW * group)
    mean = sg / n
    var = (qg / n - mean * mean).clamp_min(0.0)
    dm = dsg / n
    dvar = dqg / n + dm * (2.0 * mean.abs() + dm) + 8.0 * U64 * (qabs / n + mean * mean)
    rstd, Dr, Rr = _rstd(var, dvar, eps)

    def per_channel(t):  # [B,G] -> [B,1,1,C]
        return t.repeat_interleave(group, dim=1).view(B, 1, 1, C)

    mean, rstd, Dr, Rr, dm = (per_channel(t) for t in (mean, rstd, Dr, Rr, dm))
    g = gamma.double().to(x.device) if gamma is not None else torch.ones(C, dtype=torch.float64, device=x.device)
    be = beta.double().to(x.device) if beta is not None else torch.zeros(C, dtype=torch.float64, device=x.device)
    t = x + b - mean
    y = t * rstd * g + be
    err = (g.abs() * (t.abs() * Dr + dm * Rr) + U32 * Rr * g.abs() * x.abs()
           + 2.0 * U32 * (b.abs() + mean.abs() + dm) * Rr * g.abs() + U32 * be.abs())
    return _out(y, err, dtype, relu, residual)


def instance_norm(x: Tensor, dtype: torch.dtype, **kw) -> Tuple[Tensor, Tensor]:
    """The instance norm of x with its own sums, as pfb_instance_norm_act computes them (K from stats_k)."""
    _, H, W, C = x.shape
    s, q = sums(x)
    ds, dq = sum_errors(x, stats_k(H * W, C))
    return normalize(x, s, q, ds, dq, dtype, **kw)


def group_norm(x: Tensor, dtype: torch.dtype, group: int, **kw) -> Tuple[Tensor, Tensor]:
    """The group norm of x + bias with the sums of x, as pfb_group_norm_act computes them."""
    _, H, W, C = x.shape
    s, q = sums(x)
    ds, dq = sum_errors(x, stats_k(H * W, C))
    return normalize(x, s, q, ds, dq, dtype, group=group, **kw)


def bias_act(x: Tensor, bias: Optional[Tensor], dtype: torch.dtype, relu: bool = False,
             residual: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    x = x.double()
    y = x + bias.double().to(x.device) if bias is not None else x
    return _out(y, torch.zeros_like(y), dtype, relu, residual)


def first_conv(x: Tensor, w: Tensor, bias: Optional[Tensor], dtype: torch.dtype, relu: bool) -> Tuple[Tensor, Tensor, Tensor, Tensor, int]:
    """pfb_first_conv7x7s2 on frames x [N,H,W,3] (float64 of the stored values) with the storage-rounded filter w [64,3,7,7]:
    (ref, bound, acc, E, n) -- the output's reference and bound (epilogue RELU or LINEAR), the pre-activation acc = conv + bias
    and its accumulator bound E (both [N,H/2,W/2,64]) for the statistics, n the terms per output."""
    acc, S, n = R.conv_terms([x], w, bias, stride=2)
    E = (n + R.C_SPARE) * R.U * S
    ref, bound = R.epilogue(R.RELU if relu else R.LINEAR, acc, S, n, dtype)["out"]
    return ref, bound, acc, E, n


def split_flow(flow: Tensor, dtype: torch.dtype) -> Tuple[Tensor, Tensor]:
    """The hi / lo halves of an fp32 flow, as convf1's loaders make them (float64 of the storage-type values)."""
    f = flow.float()
    hi = f.to(dtype)
    lo = (f - hi.float()).to(dtype)
    return hi.double(), lo.double()


def flow_conv(flow: Tensor, w: Tensor, bias: Tensor, dtype: torch.dtype, lo: bool = True) -> Tuple[Tensor, Tensor]:
    """relu(conv7x7(flow) + bias) of pfb_flow_conv7x7 in float64 on the fp32 flow [B,H,W,2] and the storage-rounded filter w
    [128,2,7,7]; (ref, bound), [B,H,W,128].  ``lo=False`` computes what a kernel that drops the lo half would give instead (ref
    only; the bound returned is the same)."""
    f = flow.double()
    hi, lov = split_flow(flow, dtype)
    acc, _, _ = R.conv_terms([f if lo else hi], w, bias)
    _, S, n = R.conv_terms([hi, lov], torch.cat([w, w], 1), bias)
    ref, bound = R.epilogue(R.RELU, acc, S, n, dtype)["out"]
    rho_s, eta_s = SPLIT[dtype]
    sp = F.conv2d((rho_s * f.abs() + eta_s).permute(0, 3, 1, 2), w.double().abs(), padding=3).permute(0, 2, 3, 1)
    return ref, bound + (1.0 + R.RHO[dtype]) * sp


# ---- operands -------------------------------------------------------------------------------------------------------
def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(seed)


def norm_input(B: int, H: int, W: int, C: int, dtype: torch.dtype, seed: int, device="cpu", exact: bool = False) -> Tensor:
    """Activations [B,H,W,C] in the storage type whose mean and spread differ per (image, channel): |mean| / sigma from 0 to
    50 across the channels (shifted per image), sigma from 3e-3 to 3, both signs; channel 1 is constant (a different value
    per image).  ``exact``: values on the grid k / 4, |x| <= 2, so every fp32 partial sum of x and x^2 over < 2^18 pixels is
    exact."""
    g = _gen(device, seed)
    c = torch.arange(C, device=device, dtype=torch.float64)
    b = torch.arange(B, device=device, dtype=torch.float64).view(B, 1)
    ratio = 50.0 * ((7 * c + 3 * b) % C) / max(C - 1, 1)
    sign = torch.where(((c + b) % 2) == 0, 1.0, -1.0)
    if exact:
        sigma = 0.25 + 0.75 * torch.rand((B, C), generator=g, device=device, dtype=torch.float64)
        mean = sign * (ratio / 50.0) * 1.5
    else:
        sigma = 3e-3 * 1000.0 ** torch.rand((B, C), generator=g, device=device, dtype=torch.float64)
        mean = sign * ratio * sigma
    x = mean.view(B, 1, 1, C) + sigma.view(B, 1, 1, C) * torch.randn((B, H, W, C), generator=g, device=device, dtype=torch.float64)
    if C > 1:
        x[..., 1] = (0.75 * (b + 1) * torch.where(b % 2 == 0, 1.0, -1.0)).view(B, 1, 1)
    if exact:
        x = (4.0 * x).round().clamp(-8.0, 8.0) / 4.0
    return x.to(dtype)


def frames(N: int, H: int, W: int, dtype: torch.dtype, seed: int, device="cpu", exact: bool = False) -> Tensor:
    """First-convolution input [N,H,W,4] (RGB in [-1, 1], a zero fourth channel); ``exact``: on the grid k / 4."""
    g = _gen(device, seed)
    x = torch.zeros((N, H, W, 4), device=device, dtype=torch.float64)
    x[..., :3] = (0.6 * torch.randn((N, H, W, 3), generator=g, device=device, dtype=torch.float64)).clamp(-1.0, 1.0)
    if exact:
        x = (4.0 * x).round() / 4.0
    return x.to(dtype).contiguous()


def sparse_filter(cout: int, cin: int, taps: int, seed: int, device="cpu", zero_sum: bool = False) -> Tensor:
    """[cout, cin, 7, 7] with ``taps`` taps of +-1/2 or +-1/4 per output channel at random positions (where two fall on one
    position the later one replaces it).  ``zero_sum``: the taps come in +a / -a pairs within one input channel and pairs that
    meet add up, so for every (output, input) channel the taps sum to zero and a constant input cancels; sum |w| stays at
    most taps / 2 either way."""
    g = _gen(device, seed)
    w = torch.zeros((cout, cin * 49), device=device, dtype=torch.float64)
    rows = torch.arange(cout, device=device)
    for _ in range(taps // 2 if zero_sum else taps):
        mag = 0.5 ** torch.randint(1, 3, (cout,), generator=g, device=device).double()
        sgn = torch.where(torch.rand((cout,), generator=g, device=device) < 0.5, -1.0, 1.0).double()
        if zero_sum:
            ci = torch.randint(0, cin, (cout,), generator=g, device=device)
            p0 = torch.randint(0, 49, (cout,), generator=g, device=device)
            p1 = (p0 + torch.randint(1, 49, (cout,), generator=g, device=device)) % 49
            w[rows, ci * 49 + p0] += sgn * mag
            w[rows, ci * 49 + p1] -= sgn * mag
        else:
            pos = torch.randint(0, cin * 49, (cout,), generator=g, device=device)
            w[rows, pos] = sgn * mag
    return w.view(cout, cin, 7, 7)


def smooth_flow(B: int, H: int, W: int, seed: int, device="cpu") -> Tensor:
    """fp32 [B,H,W,2]: a smooth field of 100 to 400 px with a 1e-3 px texture on top -- large values whose differences
    between neighbours are what a zero-sum filter sees."""
    g = _gen(device, seed)
    yy = torch.arange(H, device=device, dtype=torch.float64).view(1, H, 1, 1)
    xx = torch.arange(W, device=device, dtype=torch.float64).view(1, 1, W, 1)
    ph = 6.283 * torch.rand((B, 1, 1, 2), generator=g, device=device, dtype=torch.float64)
    f = 250.0 + 150.0 * torch.sin(0.05 * xx + 0.03 * yy + ph)
    f = f + 1e-3 * torch.randn((B, H, W, 2), generator=g, device=device, dtype=torch.float64)
    return f.float().contiguous()


def exact_flow(B: int, H: int, W: int, dtype: torch.dtype, seed: int, device="cpu") -> Tensor:
    """fp32 [B,H,W,2] whose hi + lo split is exact: multiples of 2^-14 below 32 (at most 19 significant bits) for f16, of
    2^-8 below 32 (13 bits) for bf16.  With taps of +-1/2, +-1/4 every product is a multiple of 2^-16 (2^-10) and, with at
    most 8 taps, every partial sum stays below 2^7: fp32 adds them exactly."""
    g = _gen(device, seed)
    unit = 2.0 ** -14 if dtype == torch.float16 else 2.0 ** -8
    f = 31.0 * (2.0 * torch.rand((B, H, W, 2), generator=g, device=device, dtype=torch.float64) - 1.0)
    return ((f / unit).round() * unit).float().contiguous()


def assert_sums_equal(ws: Tensor, s: Tensor, q: Tensor, what: str = "") -> None:
    """The workspace sums [B,C,2] (fp64) equal the float64 sums s, q [B,C] bit for bit."""
    got = ws.view(s.shape[0], s.shape[1], 2).to(s.device)
    for k, (name, ref) in enumerate((("sum", s), ("sum of squares", q))):
        bad = (got[..., k] != ref).nonzero()
        if bad.shape[0]:
            i = tuple(bad[0].tolist())
            raise AssertionError(f"{what}: {bad.shape[0]} {name}s differ from the exact ones; first at (image, channel) {i}: "
                                 f"got {got[i + (k,)].item()!r}, exact {ref[i].item()!r}")


def assert_sums_within(ws: Tensor, s: Tensor, q: Tensor, ds: Tensor, dq: Tensor, what: str = "") -> float:
    """The workspace sums are within ds, dq of the float64 sums; returns max(err / bound)."""
    got = ws.view(s.shape[0], s.shape[1], 2).to(s.device)
    worst = 0.0
    for k, (name, ref, d) in enumerate((("sum", s, ds), ("sum of squares", q, dq))):
        worst = max(worst, R.assert_within(got[..., k], ref, d + 1e-300, what=f"{what} {name}"))
    return worst
