"""Conformance of the encoders' normalisation passes (pfb_instance_norm_act / _apply, pfb_group_norm_act / _apply,
pfb_bias_act) and of the two 7x7 first convolutions (pfb_first_conv7x7s2, pfb_flow_conv7x7) against the float64 references of
norm_reference.py, element by element, inside the per-element bounds derived there.

Two kinds of operands:
  * realistic: per-(image, channel) means and spreads that differ (|mean| / sigma from 0 to 50, sigma from 3e-3 to 3), a
    constant channel, values on both sides of the ReLU, residuals of both signs; the outputs (and the fp64 workspace sums)
    must lie inside their bounds.
  * dyadic: values on grids where every fp32 partial sum is exact.  The workspace sums then equal the float64 sums bit for bit
    (one dropped, duplicated or misattributed pixel shows), the convolutions' outputs equal the reference rounded once, and two
    calls give the same bits.

The norm sweep runs every channel count on grids on both sides of each pixels-per-block threshold of the statistics and the
normalise passes (1024, 8192, 65536 pixels), the 65535- and 65536-pixel grids for C in {64, 128, 256}, and RAFT's config-2
layer1 (16 x 220 x 512 x 64).  Every norm call goes through the C ABI with a workspace of its own, in place (out = x, as the
encoders call them) and out of place into a sentinel buffer with spare pixels behind it.  With PFB_PARITY_REPORT set, every
case appends its max(err / bound) as one JSON line."""
import json
import os
import zlib

import pytest
import torch

import conv_reference as R
import norm_reference as N

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = os.environ.get("PFB_PARITY_REPORT")  # optional: one JSON line of measured errors per check
HALF = [torch.float16, torch.bfloat16]
ALL = HALF + [torch.float32]
DT = {torch.float16: "f16", torch.bfloat16: "bf16", torch.float32: "f32"}
EPS = 1e-5
SPARE = 64  # pixels behind every out-of-place output


def _report(**kw):
    if not REPORT:
        return
    try:
        os.makedirs(os.path.dirname(REPORT) or ".", exist_ok=True)
        with open(REPORT, "a") as f:
            f.write(json.dumps(kw) + "\n")
    except OSError:
        pass


def _seed(*parts):
    return zlib.crc32("/".join(str(p) for p in parts).encode())


def _lib():
    from ptlflow_b200 import _lib as L

    return L


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _sentinel_out(shape, dtype):
    """(out, base): out a view of the first numel elements of a sentinel-filled buffer with SPARE pixels behind it."""
    numel = 1
    for s in shape:
        numel *= s
    base = torch.full((numel + SPARE * shape[-1],), R.SENTINEL, dtype=dtype, device=DEV)
    return base[:numel].view(shape), base


def _assert_spare_untouched(base, numel, what):
    tail = base[numel:]
    assert torch.equal(R.bits(tail), R.bits(torch.full_like(tail, R.SENTINEL))), f"{what}: pixels behind the output were written"


# ---- the normalisation passes ------------------------------------------------------------------------------------------
def _norm_call(kind, x, out, ws, relu, residual=None, bias=None, gamma=None, beta=None, group=1):
    L = _lib()
    lib = L.load()
    B, H, W, C = x.shape
    dt, st = L.dtype_code(x.dtype), L.stream_ptr(x.device)
    res = _ptr(residual)
    if kind == "instance":
        rc = lib.pfb_instance_norm_act(_ptr(x), _ptr(out), res, _ptr(ws), B, H, W, C, EPS, int(relu), dt, st)
    elif kind == "instance_apply":
        rc = lib.pfb_instance_norm_apply(_ptr(x), _ptr(out), res, _ptr(ws), B, H, W, C, EPS, int(relu), dt, st)
    elif kind in ("group", "group_apply"):
        fn = lib.pfb_group_norm_act if kind == "group" else lib.pfb_group_norm_apply
        rc = fn(_ptr(x), _ptr(out), res, _ptr(ws), _ptr(bias), _ptr(gamma), _ptr(beta), B, H, W, C, group, EPS, int(relu), dt, st)
    else:
        rc = lib.pfb_bias_act(_ptr(x), _ptr(bias), res, _ptr(out), _ptr(ws), B, H, W, C, int(relu), dt, st)
    L.check(rc, kind)


def _affine(C, seed, with_bias):
    g = torch.Generator(device=DEV).manual_seed(seed)
    bias = torch.randn(C, generator=g, device=DEV) if with_bias else None
    gamma = 1.0 + 0.5 * torch.randn(C, generator=g, device=DEV)
    beta = 0.3 * torch.randn(C, generator=g, device=DEV)
    return bias, gamma, beta


def run_norm(kind, B, H, W, C, dtype, relu, residual, inplace, exact=False, group=1, with_bias=True):
    """One call of kind ("instance", "group" or "bias") on fresh operands, checked; returns max(err / bound)."""
    sd = _seed(kind, B, H, W, C, dtype, relu, residual, inplace, exact, group, with_bias)
    x = N.norm_input(B, H, W, C, dtype, sd, DEV, exact=exact)
    xd = x.double()
    res = None
    if residual:
        g = torch.Generator(device=DEV).manual_seed(sd + 1)
        r = torch.randn((B, H, W, C), generator=g, device=DEV, dtype=torch.float64)
        res = ((4.0 * r).round().clamp(-8.0, 8.0) / 4.0 if exact else r).to(dtype)
    bias, gamma, beta = _affine(C, sd + 2, with_bias)
    if kind == "instance":
        ref, bound = N.instance_norm(xd, dtype, relu=relu, residual=res)
    elif kind == "group":
        ref, bound = N.group_norm(xd, dtype, group, bias=bias, gamma=gamma, beta=beta, relu=relu, residual=res)
    else:
        bias = torch.linspace(-1.0, 1.0, C, device=DEV)
        ref, bound = N.bias_act(xd, bias, dtype, relu=relu, residual=res)
    what = f"{kind} B={B} {H}x{W} C={C} {DT[dtype]} relu={relu} residual={residual} inplace={inplace} exact={exact} group={group}"

    ws = torch.full((B * C * 3,), float("nan"), dtype=torch.float64, device=DEV)
    call = lambda inp, out: _norm_call(kind, inp, out, ws, relu, res, bias, gamma if kind == "group" else None,  # noqa: E731
                                       beta if kind == "group" else None, group)
    if inplace:
        out = x.clone()
        call(out, out)
    else:
        out, base = _sentinel_out(x.shape, dtype)
        call(x, out)
    torch.cuda.synchronize()
    worst = R.assert_within(out, ref, bound, what=what)
    if not inplace:
        _assert_spare_untouched(base, x.numel(), what)
    if kind != "bias":
        s, q = N.sums(xd)
        if exact:
            N.assert_sums_equal(ws[: B * C * 2], s, q, what=what)
        else:
            N.assert_sums_within(ws[: B * C * 2], s, q, *N.sum_errors(xd, N.stats_k(H * W, C)), what=what)
    if exact and not inplace:
        again = torch.empty_like(out)
        call(x, again)
        torch.cuda.synchronize()
        assert torch.equal(R.bits(again), R.bits(out)), f"{what}: two calls differ"
    return worst


CHANNELS = [8, 16, 24, 32, 64, 96, 128, 160, 256, 512]
# every pixels-per-block threshold of the statistics (1024, 8192, 65536) and normalise (1024, 8192) passes from both sides,
# with a partial last block; batches of one and three
SMALL_GRIDS = [(1, 1, 1), (3, 1, 7), (3, 31, 33), (1, 32, 32), (3, 91, 90), (1, 64, 128)]
LARGE_GRIDS = [(1, 255, 257), (3, 256, 256)]
MODES = [(relu, residual, inplace) for relu in (False, True) for residual in (False, True) for inplace in (False, True)]


@pytest.mark.parametrize("dtype", ALL, ids=[DT[d] for d in ALL])
@pytest.mark.parametrize("C", CHANNELS)
def test_instance_norm_act(C, dtype):
    worst = 0.0
    for i, (B, H, W) in enumerate(SMALL_GRIDS):
        for relu, residual, inplace in MODES:
            worst = max(worst, run_norm("instance", B, H, W, C, dtype, relu, residual, inplace))
        worst = max(worst, run_norm("instance", B, H, W, C, dtype, True, i % 2 == 1, False, exact=True))
    _report(test="instance_norm_act", C=C, dtype=DT[dtype], max_err_over_bound=worst)


GROUPS = [(C, g) for C in CHANNELS for g in (8, 16) if C % g == 0]  # ms_raft_p's and ccmr's group sizes


@pytest.mark.parametrize("dtype", ALL, ids=[DT[d] for d in ALL])
@pytest.mark.parametrize("C,group", GROUPS, ids=[f"C{c}-g{g}" for c, g in GROUPS])
def test_group_norm_act(C, group, dtype):
    worst = 0.0
    for i, (B, H, W) in enumerate(SMALL_GRIDS):
        for j, (relu, residual, inplace) in enumerate(MODES):
            worst = max(worst, run_norm("group", B, H, W, C, dtype, relu, residual, inplace, group=group, with_bias=j % 2 == 0))
        worst = max(worst, run_norm("group", B, H, W, C, dtype, True, True, False, exact=True, group=group, with_bias=i % 2 == 0))
    _report(test="group_norm_act", C=C, group=group, dtype=DT[dtype], max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", ALL, ids=[DT[d] for d in ALL])
@pytest.mark.parametrize("C", CHANNELS)
def test_bias_act(C, dtype):
    worst = 0.0
    for B, H, W in SMALL_GRIDS:
        for relu, residual, inplace in MODES:
            worst = max(worst, run_norm("bias", B, H, W, C, dtype, relu, residual, inplace))
    _report(test="bias_act", C=C, dtype=DT[dtype], max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", ALL, ids=[DT[d] for d in ALL])
@pytest.mark.parametrize("kind", ["instance", "group", "bias"])
@pytest.mark.parametrize("C", [64, 128, 256])
def test_norm_large_grids(C, kind, dtype):
    """65535 and 65536 pixels: the statistics pass's largest pixels-per-block step, from both sides."""
    worst = 0.0
    for B, H, W in LARGE_GRIDS:
        kw = dict(group=16) if kind == "group" else {}
        worst = max(worst, run_norm(kind, B, H, W, C, dtype, True, True, True, **kw))
        worst = max(worst, run_norm(kind, B, H, W, C, dtype, False, False, False, **kw))
        if kind != "bias":
            worst = max(worst, run_norm(kind, B, H, W, C, dtype, True, False, False, exact=True, **kw))
    _report(test="norm_large_grids", kind=kind, C=C, dtype=DT[dtype], max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", ALL, ids=[DT[d] for d in ALL])
@pytest.mark.parametrize("kind", ["instance", "group", "bias"])
def test_norm_config2_layer1(kind, dtype):
    """RAFT's layer1 at 1024 x 436 (padded to 440) for 16 frames: 16 x 220 x 512 x 64, in place as the encoders call it; the
    dyadic case's sums must match bit for bit at this size too."""
    kw = dict(group=8) if kind == "group" else {}
    worst = run_norm(kind, 16, 220, 512, 64, dtype, True, True, True, **kw)
    if kind != "bias":
        worst = max(worst, run_norm(kind, 16, 220, 512, 64, dtype, True, False, False, exact=True, **kw))
    _report(test="norm_config2_layer1", kind=kind, dtype=DT[dtype], max_err_over_bound=worst)


# ---- pfb_first_conv7x7s2 ---------------------------------------------------------------------------------------------------
FC_SHAPES = [
    (1, 2, 8),        # the minimum: one output row, four pixels
    (3, 6, 18),       # odd Ho: the last pair's second row is outside
    (2, 20, 258),     # a one-pixel second 128-pixel segment
    (1, 8, 512),      # exactly two segments
    (13, 42, 200),    # 11 work items per image: CTAs whose items straddle two images
    (16, 440, 1024),  # RAFT config 2: several items per CTA
]
FC_MODES = {"stats": (False, False, True), "stats_bias_relu": (True, True, True), "bias_relu": (True, True, False)}


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _first_conv_operands(N_, H, W, dtype, exact, sd):
    x = N.frames(N_, H, W, dtype, sd, DEV, exact=exact)
    g = torch.Generator(device=DEV).manual_seed(sd + 1)
    if exact:
        w = N.sparse_filter(64, 3, 6, sd + 2, DEV)
        bias = (16.0 * torch.rand(64, generator=g, device=DEV) - 8.0).round() / 16.0
    else:
        w = 0.12 * torch.randn((64, 3, 7, 7), generator=g, device=DEV, dtype=torch.float64)
        bias = 0.5 * torch.randn(64, generator=g, device=DEV)
    return x, R.q(w, dtype), bias.float()


def run_first_conv(N_, H, W, dtype, mode, exact):
    from ptlflow_b200 import ops

    L = _lib()
    with_bias, relu, with_stats = FC_MODES[mode]
    sd = _seed("first_conv", N_, H, W, dtype, mode, exact)
    x, wq, bias = _first_conv_operands(N_, H, W, dtype, exact, sd)
    b = bias if with_bias else None
    ref, bound, acc, E, _ = N.first_conv(x[..., :3].double(), wq, b.double() if b is not None else None, dtype, relu)
    wpack = ops.pack_first_conv(wq.float(), dtype).to(DEV)
    Ho, Wo = H // 2, W // 2
    what = f"first_conv {N_}x{H}x{W} {DT[dtype]} {mode} exact={exact}"

    def call():
        out, base = _sentinel_out((N_, Ho, Wo, 64), dtype)
        ws = torch.zeros(N_ * 64 * 2, dtype=torch.float64, device=DEV) if with_stats else None
        L.check(L.load().pfb_first_conv7x7s2(_ptr(x), _ptr(wpack), _ptr(b), _ptr(out), _ptr(ws), N_, H, W, int(relu),
                                             L.dtype_code(dtype), L.stream_ptr(DEV)), "first_conv7x7s2")
        torch.cuda.synchronize()
        return out, base, ws

    out, base, ws = call()
    worst = R.assert_within(out, ref, bound, what=what)
    _assert_spare_untouched(base, out.numel(), what)
    if exact:
        assert torch.equal(R.bits(out), R.bits(ref.to(dtype))), f"{what}: not the reference rounded once"
    s, q = N.sums(acc)
    if with_stats:
        if exact:
            N.assert_sums_equal(ws, s, q, what=what)
        else:
            _, per_cta = N.first_conv_items(N_, Ho, Wo, _sms())
            worst = max(worst, N.assert_sums_within(ws, s, q, *N.conv_sum_errors(acc, E, N.first_conv_k(per_cta)), what=what))
    if exact:
        out2, _, ws2 = call()
        assert torch.equal(R.bits(out2), R.bits(out)), f"{what}: two calls differ"
        if with_stats:
            assert torch.equal(ws2, ws), f"{what}: two calls give different sums"
    if mode == "stats" and not exact:
        worst = max(worst, _chain(out, ws, acc, E, dtype, what))
    return worst


def _chain(y, ws, acc, E, dtype, what):
    """instance_norm_apply (in place, as the encoders chain it) and group_norm_apply (bias folded, affine) fed by the first
    convolution's sums; the reference normalises the stored output with the statistics of the exact convolution."""
    N_, Ho, Wo, C = y.shape
    _, per_cta = N.first_conv_items(N_, Ho, Wo, _sms())
    s, q = N.sums(acc)
    ds, dq = N.conv_sum_errors(acc, E, N.first_conv_k(per_cta))
    yd = y.double()
    wsf = torch.cat([ws, torch.full((N_ * C,), float("nan"), dtype=torch.float64, device=DEV)])
    bias, gamma, beta = _affine(C, _seed(what, "chain"), True)
    worst = 0.0
    for group in (8, 16):
        out = torch.empty_like(y)
        _norm_call("group_apply", y, out, wsf, True, bias=bias, gamma=gamma, beta=beta, group=group)
        torch.cuda.synchronize()
        ref, bound = N.normalize(yd, s, q, ds, dq, dtype, relu=True, bias=bias, gamma=gamma, beta=beta, group=group)
        worst = max(worst, R.assert_within(out, ref, bound, what=f"{what} -> group_norm_apply group={group}"))
    ref, bound = N.normalize(yd, s, q, ds, dq, dtype, relu=True)
    _norm_call("instance_apply", y, y, wsf, True)
    torch.cuda.synchronize()
    return max(worst, R.assert_within(y, ref, bound, what=f"{what} -> instance_norm_apply"))


@pytest.mark.parametrize("dtype", HALF, ids=[DT[d] for d in HALF])
@pytest.mark.parametrize("mode", list(FC_MODES))
@pytest.mark.parametrize("n,h,w", FC_SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in FC_SHAPES])
def test_first_conv7x7s2(n, h, w, mode, dtype):
    worst = run_first_conv(n, h, w, dtype, mode, exact=False)
    if h * w // 4 <= 29000:  # dyadic sums stay exact (config 2 is checked against the bound only)
        worst = max(worst, run_first_conv(n, h, w, dtype, mode, exact=True))
    _report(test="first_conv7x7s2", shape=[n, h, w], mode=mode, dtype=DT[dtype], max_err_over_bound=worst)


def test_first_conv_ctas_straddle_images():
    """At (13, 42, 200) the work items of some CTA belong to two images, so the epilogue flushes its sums mid-run."""
    n_items, per_cta = N.first_conv_items(13, 21, 100, _sms())
    per_img = n_items // 13
    straddle = [k for k in range(0, n_items, per_cta) if k // per_img != (min(k + per_cta, n_items) - 1) // per_img]
    assert per_cta > 1 and straddle, (n_items, per_cta)


# ---- pfb_flow_conv7x7 (convf1) --------------------------------------------------------------------------------------------
FL_SHAPES = [(1, 1, 1), (2, 1, 130), (3, 7, 128), (2, 11, 129), (1, 55, 128), (8, 55, 128)]
FL_LAYOUTS = [(128, 0), (160, 16)]  # (out_stride, out_offset): the loop's motion-feature buffer, and a wider strided one
FLOWS = ["zero", "tiny", "large", "smooth", "exact"]


def _flow_operands(kind, B, H, W, dtype, sd):
    g = torch.Generator(device=DEV).manual_seed(sd)
    bias = 0.3 * torch.randn(128, generator=g, device=DEV)
    w = 0.1 * torch.randn((128, 2, 7, 7), generator=g, device=DEV, dtype=torch.float64)
    if kind == "zero":
        flow = torch.zeros((B, H, W, 2), device=DEV)
    elif kind == "tiny":  # the f16 lo half is subnormal
        flow = 1e-4 * torch.randn((B, H, W, 2), generator=g, device=DEV)
    elif kind == "large":
        flow = 400.0 * (2.0 * torch.rand((B, H, W, 2), generator=g, device=DEV) - 1.0)
    elif kind == "smooth":
        flow = N.smooth_flow(B, H, W, sd + 1, DEV)
        w = N.sparse_filter(128, 2, 6, sd + 2, DEV, zero_sum=True)
    else:
        flow = N.exact_flow(B, H, W, dtype, sd + 1, DEV)
        w = N.sparse_filter(128, 2, 6, sd + 2, DEV)
        bias = (16.0 * torch.rand(128, generator=g, device=DEV) - 8.0).round() / 16.0
    return flow.contiguous(), R.q(w, dtype), bias.float()


@pytest.mark.parametrize("dtype", HALF, ids=[DT[d] for d in HALF])
@pytest.mark.parametrize("b,h,w", FL_SHAPES, ids=[f"{b}x{h}x{w}" for b, h, w in FL_SHAPES])
def test_flow_conv7x7(b, h, w, dtype):
    from ptlflow_b200 import ops

    worst = {}
    for kind in FLOWS:
        sd = _seed("flow_conv", b, h, w, dtype, kind)
        flow, wq, bias = _flow_operands(kind, b, h, w, dtype, sd)
        ref, bound = N.flow_conv(flow, wq, bias.double(), dtype)
        wpack = ops.pack_flow_conv(wq.float(), dtype).to(DEV)
        for stride, off in FL_LAYOUTS:
            what = f"flow_conv {b}x{h}x{w} {DT[dtype]} {kind} stride={stride} offset={off}"
            outs = []
            for _ in range(2 if kind == "exact" else 1):
                out, base = _sentinel_out((b, h, w, stride), dtype)
                before = out.clone()
                ops.flow_conv7x7(flow, wpack, bias, out, out_offset=off)
                torch.cuda.synchronize()
                got = out[..., off:off + 128]
                worst[kind] = max(worst.get(kind, 0.0), R.assert_within(got, ref, bound, what=what))
                R.assert_untouched(out, before, off, off + 128, what=what)
                _assert_spare_untouched(base, out.numel(), what)
                outs.append(got)
            if kind == "exact":
                assert torch.equal(R.bits(outs[0]), R.bits(ref.to(dtype))), f"{what}: not the reference rounded once"
                assert torch.equal(R.bits(outs[1]), R.bits(outs[0])), f"{what}: two calls differ"
    for kind, v in worst.items():
        _report(test="flow_conv7x7", shape=[b, h, w], flow=kind, dtype=DT[dtype], max_err_over_bound=v)


# ---- argument checks -------------------------------------------------------------------------------------------------------
def _declined(fn, *args, match):
    L = _lib()
    lib = L.load()
    torch.cuda.synchronize()
    n0 = lib.pfb_launch_count(-1)
    with pytest.raises(RuntimeError, match=match):
        L.check(fn(*args), "call")
    torch.cuda.synchronize()
    assert lib.pfb_launch_count(-1) == n0


def test_bad_arguments_raise_before_any_launch():
    L = _lib()
    lib = L.load()
    st, f16 = L.stream_ptr(DEV), L.dtype_code(torch.float16)
    buf = torch.zeros(1 << 20, dtype=torch.float16, device=DEV)
    ws = torch.full((1 << 16,), float("nan"), dtype=torch.float64, device=DEV)
    p, w = buf.data_ptr(), ws.data_ptr()
    for C in (12, 520):
        _declined(lib.pfb_instance_norm_act, p, p, None, w, 1, 4, 4, C, EPS, 1, f16, st, match="multiple of 8")
        _declined(lib.pfb_instance_norm_apply, p, p, None, w, 1, 4, 4, C, EPS, 1, f16, st, match="multiple of 8")
        _declined(lib.pfb_group_norm_act, p, p, None, w, None, None, None, 1, 4, 4, C, 4, EPS, 1, f16, st, match="multiple of 8")
        _declined(lib.pfb_bias_act, p, None, None, p, w, 1, 4, 4, C, 1, f16, st, match="multiple of 8")
    assert torch.isnan(ws).all(), "a declined call touched the workspace"
    for fn in (lib.pfb_group_norm_act, lib.pfb_group_norm_apply):
        _declined(fn, p, p, None, w, None, None, None, 1, 4, 4, 64, 3, EPS, 1, f16, st, match="must divide")
        _declined(fn, p, p, None, w, None, None, None, 1, 4, 4, 64, 0, EPS, 1, f16, st, match="must divide")
    wpack = torch.zeros(1 << 16, dtype=torch.float16, device=DEV).data_ptr()
    for (n, h, wd), dt in (((1, 7, 16), f16), ((1, 8, 17), f16), ((1, 8, 6), f16), ((1, 8, 16), L.dtype_code(torch.float32))):
        _declined(lib.pfb_first_conv7x7s2, p, wpack, None, p, None, n, h, wd, 1, dt, st, match="first_conv7x7s2")
    flow = torch.zeros((1, 4, 8, 2), device=DEV).data_ptr()
    _declined(lib.pfb_flow_conv7x7, flow, wpack, w, p, 136, 4, 1, 4, 8, f16, st, match="multiples of 8")
