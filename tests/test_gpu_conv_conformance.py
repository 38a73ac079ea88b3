"""Conformance of the implicit-GEMM convolution (pfb_conv2d) against the float64 reference of conv_reference.py, element by
element, across the wgmma kernel's tiling, pipeline and epilogue space.

Every case runs the wgmma kernel (impl = 2, so a silent fallback cannot hide a path) on f16 and bf16, and the SIMT kernel
(impl = 1) on f16, bf16 and fp32.  Each case reaches its path by its shape alone (the planner in conv_umma.cu:
plan_conv_umma); test_trace_covers_every_path checks from the launch trace that the sweep as a whole reaches every halo
mode, weight-stage grouping, N tile width, the two-stage rings, CTAs with several work items and every epilogue.  Output
buffers start as a sentinel: columns outside the layer's output range (the pad columns of Cout_pad_k among them) must keep
it.  With PFB_PARITY_REPORT set, every case appends its max(err / bound) as one JSON line."""
import json
import os
import subprocess
import sys
import zlib

import pytest
import torch

import conv_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = os.environ.get("PFB_PARITY_REPORT")  # optional: one JSON line of measured errors per check
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF = [torch.float16, torch.bfloat16]


def _report(**kw):
    if not REPORT:
        return
    try:
        os.makedirs(os.path.dirname(REPORT), exist_ok=True)
        with open(REPORT, "a") as f:
            f.write(json.dumps(kw) + "\n")
    except OSError:
        pass


def case(name, B, H, W, k, srcs, cout, epi, wgmma=True, simt=True, **kw):
    """srcs: (channels,) or (channels, stride, offset) per source.  kw: scale, hidden, out_offset, residual=(stride, offset),
    post, addend=stride, per_sample."""
    srcs = [s if len(s) == 3 else (s[0], (s[0] + 7) // 8 * 8, 0) for s in srcs]
    return dict(name=name, B=B, H=H, W=W, KH=k[0], KW=k[1], srcs=srcs, cout=cout, epi=epi, wgmma=wgmma, simt=simt, **kw)


CASES = [
    # halo 0, TW 32 x TH 4; partial M tiles in x (90 of 96) and y (41 of 44); three sources, two of them at an offset inside
    # a wider pixel stride and one ending in an 8-channel chunk; out_offset 16
    case("halo0_tw32_three_src", 3, 41, 90, (3, 3), [(40, 64, 8), (64,), (72, 88, 16)], 96, R.LINEAR, scale=-0.625, out_offset=16),
    case("halo1_bgroup3", 1, 55, 128, (3, 3), [(64,)], 64, R.RELU),
    # halo 1, all five taps of a patch in one weight stage; partial x tile (200 of 256); Cout % 32 == 30 with the flow columns
    case("halo1_bgroup5_append_flow", 2, 3, 200, (1, 5), [(100, 104, 0)], 62, R.LINEAR_APPEND_FLOW, out_offset=8),
    case("halo2_tw16", 1, 55, 128, (7, 1), [(128,)], 128, R.GELU),
    # plain epilogue: the output staging tile leaves room for two activation and two weight stages only
    case("two_weight_stages", 1, 6, 128, (5, 1), [(128,)], 128, R.RELU),
    case("nt32_x5", 1, 55, 128, (1, 1), [(96,)], 160, R.LINEAR, scale=1.5),                 # n_work 275 > 132 CTAs
    case("nt64_x5_staged", 2, 20, 64, (3, 3), [(64,)], 320, R.GELU),
    case("nt96_x2_direct", 1, 55, 128, (1, 1), [(64,), (48, 56, 8)], 192, R.RELU, out_offset=8),
    case("nt128_x8_staged", 1, 55, 128, (1, 1), [(64,)], 1024, R.LINEAR, scale=0.5),        # n_work 440
    case("gru_zr_hd128", 4, 55, 128, (3, 3), [(128,), (128,), (128,)], 256, R.GRU_ZR, hidden=128),  # NT 128 x 2, n_work 440
    case("gru_q_hd128", 4, 55, 128, (3, 3), [(128,), (128,), (128,)], 128, R.GRU_Q, hidden=128),
    case("gru_zr_hd96", 2, 11, 21, (1, 5), [(96,), (64,)], 192, R.GRU_ZR, hidden=96),
    case("gru_q_hd96", 2, 11, 21, (1, 5), [(96,), (64,)], 96, R.GRU_Q, hidden=96),
    case("gru_zr_hd64", 1, 13, 19, (5, 1), [(64,), (32,)], 128, R.GRU_ZR, hidden=64, out_offset=8),
    case("gru_q_hd64", 1, 13, 19, (5, 1), [(64,), (32,)], 64, R.GRU_Q, hidden=64),
    case("axpy", 2, 17, 33, (1, 1), [(128,)], 64, R.AXPY, hidden=72, scale=0.3),
    # the GMA aggregate's form: one weight matrix per sample (rows b * w_rows_per_sample of weight_k); wgmma only
    case("axpy_per_sample", 3, 9, 40, (1, 1), [(96,)], 64, R.AXPY, hidden=64, scale=-0.5, per_sample=True, simt=False),
    # per-pixel addend instead of the bias (stride 136 > Cout_pad_k); wgmma only
    case("gru_zr_addend", 2, 10, 30, (3, 3), [(64,)], 128, R.GRU_ZR, hidden=64, addend=136, simt=False),
    case("linear_f32", 2, 9, 20, (3, 3), [(128,)], 48, R.LINEAR_F32, scale=0.5, out_offset=8),
    case("residual_gelu", 2, 9, 20, (1, 1), [(192,)], 256, R.RESIDUAL_GELU, residual=(320, 32)),
    case("residual_gelu_post", 2, 9, 20, (3, 3), [(192,)], 128, R.RESIDUAL_GELU, residual=(200, 64), post=True),
    case("relu_append_flow_126", 2, 11, 21, (3, 3), [(256,)], 126, R.RELU_APPEND_FLOW),
    # APPEND_FLOW with Cout % 32 in {0, 31}: the wgmma kernel declines them (auto selection takes the SIMT kernel)
    case("relu_append_flow_128", 1, 6, 40, (3, 3), [(64,)], 128, R.RELU_APPEND_FLOW, wgmma=False),
    case("relu_append_flow_95", 1, 6, 40, (3, 3), [(64,)], 95, R.RELU_APPEND_FLOW, wgmma=False),
    case("linear_append_flow_64", 1, 6, 40, (1, 1), [(64,)], 64, R.LINEAR_APPEND_FLOW, wgmma=False),
    case("linear_append_flow_127", 1, 6, 40, (1, 1), [(64,)], 127, R.LINEAR_APPEND_FLOW, wgmma=False),
    # grids smaller than the kernel
    case("grid_1x1_k3x3", 1, 1, 1, (3, 3), [(64,)], 64, R.RELU),
    case("grid_2x3_k5x5", 2, 2, 3, (5, 5), [(40,)], 32, R.LINEAR, scale=2.0),
]
BY_NAME = {c["name"]: c for c in CASES}


def _seed(*parts):
    return zlib.crc32("/".join(str(p) for p in parts).encode())


def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV) * scale


class _Conv(torch.nn.Module):
    """A weight / bias holder in nn.Conv2d's layout for ops.PackedConv."""

    def __init__(self, weight, bias):
        super().__init__()
        self.weight, self.bias = weight, bias


def run(c, dtype, impl, out_misalign=False, aux_misalign=False, declined=False):
    """Runs case c once and checks it.  Returns max(err / bound) over its outputs.  ``declined``: the call must raise instead,
    without launching anything."""
    from ptlflow_b200 import _lib, ops

    B, H, W, KH, KW, epi, cout = c["B"], c["H"], c["W"], c["KH"], c["KW"], c["epi"], c["cout"]
    name, hd = c["name"], c.get("hidden", 0)
    chans = [s[0] for s in c["srcs"]]
    cin = sum(chans)
    sd = _seed(name)
    # sources: NaN everywhere outside [offset, offset + channels) -- pad columns and the channels of other layers
    srcs, xs = [], []
    for i, (ch, stride, off) in enumerate(c["srcs"]):
        t = torch.full((B, H, W, stride), float("nan"), dtype=dtype, device=DEV)
        t[..., off:off + ch] = _randn((B, H, W, ch), sd + i).to(dtype)
        srcs.append((t, ch, off))
        xs.append(t[..., off:off + ch].double())
    w = _randn((cout, cin, KH, KW), sd + 10, (cin * KH * KW) ** -0.5)
    bias = _randn((cout,), sd + 11, 0.1)
    packed = ops.PackedConv([_Conv(w, bias)], dtype, DEV, src_channels=chans)
    wq = R.q(w, dtype)
    kw = dict(epilogue=epi, impl=impl, scale=c.get("scale", 1.0), hidden=hd)
    ref_kw = dict(scale=kw["scale"], hidden=hd)
    addend = None
    per_sample = c.get("per_sample", False)
    if per_sample:  # sample b's matrix at rows [b * rows, b * rows + Cout_pad_k) of weight_k; the rows between are never read
        rows = packed.Cout_pad_k + 32
        wk = torch.full((B, rows, packed.Cin_pad), float("nan"), dtype=dtype, device=DEV)
        wk[:, :packed.Cout_pad_k] = 0
        wps = _randn((B, cout, cin), sd + 12, cin ** -0.5).to(dtype)
        wk[:, :cout, :cin] = wps
        packed.weight_k = wk
        kw["w_rows_per_sample"] = rows
        wq = wps.double()
    if c.get("addend"):
        add_t = _randn((B, H, W, c["addend"]), sd + 13).to(dtype)
        kw["addend"] = add_t
        addend = add_t[..., :cout].double()
    acc, S, n = R.conv_terms(xs, wq, bias.double(), addend, per_sample=per_sample)

    out_dtype = torch.float32 if epi == R.LINEAR_F32 else dtype
    append = epi in (R.RELU_APPEND_FLOW, R.LINEAR_APPEND_FLOW)
    ncols = hd if epi == R.GRU_ZR else (cout + 2 if append else cout)
    off = c.get("out_offset", 0)
    out_stride = (off + max(ncols, packed.Cout_pad_k if dtype != torch.float32 else cout) + 8 + 7) // 8 * 8
    numel = B * H * W * out_stride
    base = torch.full((numel + 8,), R.SENTINEL, dtype=out_dtype, device=DEV)
    out = base[1:numel + 1] if out_misalign else base[:numel]  # 2 bytes past a 16-byte boundary, or aligned
    out = out.view(B, H, W, out_stride)
    before = out.clone()
    aux = {}
    if epi in (R.GRU_ZR, R.GRU_Q, R.AXPY):
        hs = torch.tanh(_randn((B, H, W, hd), sd + 14)).to(dtype)
        if aux_misalign:
            hb = torch.empty(hs.numel() + 8, dtype=dtype, device=DEV)
            hb[1:hs.numel() + 1] = hs.flatten()
            hs = hb[1:hs.numel() + 1].view(B, H, W, hd)
        kw["aux_h"] = hs
        ref_kw["h"] = hs.double()
    if epi in (R.GRU_ZR, R.GRU_Q):
        zs = torch.full((B, H, W, hd), R.SENTINEL, dtype=dtype, device=DEV)
        if epi == R.GRU_Q:
            zs = torch.sigmoid(_randn((B, H, W, hd), sd + 15)).to(dtype)
            ref_kw["z"] = zs.double()
        kw["aux_z"] = zs
    if epi == R.RESIDUAL_GELU:
        rstride, roff = c["residual"]
        res = _randn((B, H, W, rstride), sd + 16).to(dtype)
        kw["residual"] = (res, roff)
        ref_kw["residual"] = res[..., roff:roff + cout].double()
        if c.get("post"):
            kw["post_w"], kw["post_b"] = _randn((cout,), sd + 17, 0.5), _randn((cout,), sd + 18, 0.1)
            ref_kw["post_w"], ref_kw["post_b"] = kw["post_w"].double(), kw["post_b"].double()
    if append:
        kw["flow"] = _randn((B, H, W, 2), sd + 19, 3.0)
        ref_kw["flow"] = kw["flow"].double()

    if declined:
        lib = _lib.load()
        torch.cuda.synchronize()
        n0 = lib.pfb_launch_count(-1)
        with pytest.raises(RuntimeError, match="wgmma path does not support"):
            ops.conv2d(srcs, packed, out, out_offset=off, **kw)
        torch.cuda.synchronize()
        assert lib.pfb_launch_count(-1) == n0
        assert torch.equal(R.bits(out), R.bits(before))
        return None
    ops.conv2d(srcs, packed, out, out_offset=off, **kw)
    torch.cuda.synchronize()
    refs = R.epilogue(epi, acc, S, n, out_dtype, **ref_kw)
    what = f"{name} {dtype} impl={impl}"
    worst = R.assert_within(out[..., off:off + ncols], *refs["out"], what=what)
    R.assert_untouched(out, before, off, off + ncols, what=what)
    if epi == R.GRU_ZR:
        worst = max(worst, R.assert_within(kw["aux_z"], *refs["z"], what=what + " z"))
    return worst


def _variants(c):
    v = []
    if c["wgmma"]:
        v += [(dt, 2) for dt in HALF]
    else:
        v += [(dt, 0) for dt in HALF]  # declined by the wgmma kernel: auto selection must give the SIMT result
    if c["simt"]:
        v += [(dt, 1) for dt in HALF + [torch.float32]]
    return v


PARAMS = [pytest.param(c["name"], dt, impl, id=f"{c['name']}-{str(dt)[6:]}-impl{impl}") for c in CASES for dt, impl in _variants(c)]


@pytest.mark.parametrize("name,dtype,impl", PARAMS)
def test_conv_conformance(name, dtype, impl):
    worst = run(BY_NAME[name], dtype, impl)
    _report(test="conv_conformance", case=name, dtype=str(dtype), impl=impl, max_err_over_bound=worst)


def run_wgmma_sweep():
    """Every wgmma case once per half type (test_trace_covers_every_path runs this in a subprocess with the launch trace on)."""
    for c in CASES:
        if c["wgmma"]:
            for dt in HALF:
                run(c, dt, 2)


# vertical kernels whose preferred vertical-halo tile leaves no room for two weight stages (64-wide tiles on short grids)
TALL = [(kh, h, w, cout) for kh in (7, 9, 11, 13, 15) for h, w, cout in ((6, 128, 128), (2, 200, 256), (6, 64, 64))]


@pytest.mark.parametrize("kh,h,w,cout", TALL)
@pytest.mark.parametrize("dtype", HALF, ids=["float16", "bfloat16"])
def test_tall_vertical_kernels(kh, h, w, cout, dtype):
    """impl 0 used to fail with "unsupported" here after the wgmma predicate had accepted the shape; now the planner takes a
    narrower vertical tile (or no halo) and both auto selection and the wgmma kernel itself compute the layer."""
    c = case(f"tall_{kh}x1_{h}x{w}_{cout}", 1, h, w, (kh, 1), [(128,)], cout, R.RELU)
    for impl in (0, 2):
        worst = run(c, dtype, impl)
        _report(test="conv_conformance", case=c["name"], dtype=str(dtype), impl=impl, max_err_over_bound=worst)


def _declined(c, dtype, **mis):
    """impl 2 raises without launching anything; impl 0 computes the layer on the SIMT kernel."""
    run(c, dtype, 2, declined=True, **mis)
    worst = run(c, dtype, 0, **mis)
    _report(test="conv_conformance", case=c["name"] + "_declined", dtype=str(dtype), impl=0, max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", HALF, ids=["float16", "bfloat16"])
@pytest.mark.parametrize("name", ["relu_append_flow_128", "relu_append_flow_95", "linear_append_flow_64", "linear_append_flow_127"])
def test_append_flow_cout_declined(name, dtype):
    """The wgmma epilogue can place the flow columns only after a last chunk with room for both (Cout % 32 in 1..30)."""
    _declined(BY_NAME[name], dtype)


@pytest.mark.parametrize("dtype", HALF, ids=["float16", "bfloat16"])
def test_misaligned_out_declined(dtype):
    _declined(case("misaligned_out", 1, 7, 30, (3, 3), [(64,)], 64, R.RELU), dtype, out_misalign=True)


@pytest.mark.parametrize("dtype", HALF, ids=["float16", "bfloat16"])
@pytest.mark.parametrize("epi", [R.GRU_Q, R.AXPY], ids=["gru_q", "axpy"])
def test_misaligned_aux_declined(epi, dtype):
    _declined(case("misaligned_aux", 1, 7, 30, (1, 1), [(64,)], 64, epi, hidden=64), dtype, aux_misalign=True)


@pytest.mark.parametrize("what", ["four_sources", "fp32_source", "cout_16"])
def test_wgmma_declines_without_launch(what):
    """Shapes the wgmma predicate declines: impl 2 raises before any launch, impl 0 gives the SIMT result."""
    from ptlflow_b200 import _lib, ops

    dtype = torch.float16
    if what == "four_sources":
        _declined(case("four_sources", 1, 5, 24, (3, 3), [(64,), (32,), (16,), (64,)], 64, R.RELU), dtype)
        return
    if what == "cout_16":
        _declined(case("cout_16", 2, 5, 24, (3, 3), [(64,)], 16, R.LINEAR, scale=0.5), dtype)
        return
    # an fp32 source (e.g. the flow) next to a half-precision one
    B, H, W = 1, 5, 24
    x = _randn((B, H, W, 64), 1).to(dtype)
    f = _randn((B, H, W, 8), 2)
    w = _randn((64, 72, 3, 3), 3, 72 ** -0.5)
    bias = _randn((64,), 4, 0.1)
    packed = ops.PackedConv([_Conv(w, bias)], dtype, DEV, src_channels=[64, 8])
    lib = _lib.load()
    out = torch.full((B, H, W, 64), R.SENTINEL, dtype=dtype, device=DEV)
    torch.cuda.synchronize()
    n0 = lib.pfb_launch_count(-1)
    with pytest.raises(RuntimeError, match="wgmma path does not support"):
        ops.conv2d([x, f], packed, out, R.RELU, impl=2)
    torch.cuda.synchronize()
    assert lib.pfb_launch_count(-1) == n0
    ops.conv2d([x, f], packed, out, R.RELU, impl=0)
    acc, S, n = R.conv_terms([x.double(), f.double()], R.q(w, dtype), bias.double())
    R.assert_within(out, *R.epilogue(R.RELU, acc, S, n, dtype)["out"], what="fp32 source")


def test_trace_covers_every_path(tmp_path):
    """The wgmma sweep, run once with PFB_CONV_TRACE, reaches every halo mode, weight-stage grouping, N tile width, the
    two-stage rings, CTAs with several work items and every epilogue but FLOW (which has its own kernels)."""
    trace = tmp_path / "conv_trace.jsonl"
    env = dict(os.environ, PFB_CONV_TRACE=str(trace))
    env.pop("PFB_PARITY_REPORT", None)
    code = ("import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; import test_gpu_conv_conformance as T; T.run_wgmma_sweep()")
    r = subprocess.run([sys.executable, "-c", code, ROOT, os.path.join(ROOT, "tests")], env=env, cwd=str(tmp_path),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    plans = [json.loads(line) for line in trace.read_text().splitlines() if line.strip()]
    assert len(plans) == 2 * sum(c["wgmma"] for c in CASES)
    seen = lambda key: {p[key] for p in plans}  # noqa: E731
    assert {0, 1, 2} <= seen("halo")
    assert {1, 3, 5} <= seen("b_group")
    assert {32, 64, 96, 128} <= seen("NT")
    assert any(p["a_stages"] == 2 and p["b_stages"] == 2 for p in plans)
    assert any(p["n_work"] > 2 * p["grid"] for p in plans)
    assert set(R.EPI_NAMES) <= seen("epi"), sorted(set(R.EPI_NAMES) - seen("epi"))
    # the named shapes reach their paths
    by = {}
    for p in plans:
        by.setdefault((p["KH"], p["KW"], p["halo"], p["TW"], p["TH"], p["NT"], p["b_group"]), p)
    assert (3, 3, 0, 32, 4, 96, 1) in by
    assert (3, 3, 1, 128, 1, 64, 3) in by
    assert (1, 5, 1, 128, 1, 64, 5) in by
    assert (7, 1, 2, 16, 8, 128, 1) in by
