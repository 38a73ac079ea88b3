"""Conformance of the correlation kernels (volume, pyramid, lookup, on-the-fly lookup, feature pooling) against the float64
reference of corr_reference.py, element by element, across their layouts, tiles and on-the-fly regions.

* Volume: the dense wgmma kernel (impl = 2, so a silent fallback cannot hide a path) on f16 / bf16 and the SIMT kernel
  followed by avg_pool2x2 (impl = 1) on f16 / bf16 / fp32, over C = 64 .. 256 (two B stages at C <= 128, one above; level 0
  through the TMA store when W % 8 == 0 and C <= 192, and once more with PFB_VOLUME_TMA_STORE=0 through the direct vector
  stores), odd H, grids smaller than one 8 x 16 patch, 1 .. 4 levels, B > 1, N not a multiple of 128, several patch groups
  and one (B = 5 at 55 x 128).  The tiled (T84) kernel on the same shapes and on target grids of their own.  Every level
  starts as the sentinel and sits between guard elements that must keep it; the pad of the tiled levels must be zero
  where the kernel writes it (all of level 0; on levels 1-3 the pad columns of the stored row chunks).
* Lookup from stored levels: the radius 3 / 4 fast path, the generic kernel (NCHW, r = 5), level_hw, and every (R, L) the
  tiled kernel instantiates, on coordinates with integers, x = W - 1, -1e-7, -40, NaN, +-inf, values either side of 1e7 at
  every level and windows starting at every tile column; outputs inside a sentinel buffer with pad columns, tiled pads
  poisoned with 1000 and with NaN.
* On the fly: the tensor-core kernel (+ its SIMT pass for flagged queries) and the SIMT kernel on f16 / bf16, fp32 on the
  SIMT kernel, C = 64 .. 256 and 96 channels padded to 128 with scale 1/sqrt(96).  The flags must equal otf_plan's, and
  the band counts the kernel records under PFB_OTF_TRACE must equal otf_plan's.
* Calls the kernels refuse raise without launching anything.
With PFB_PARITY_REPORT set, every case appends its max(err / bound) as one JSON line."""
import json
import math
import os
import subprocess
import sys
import zlib

import pytest
import torch

import corr_reference as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = os.environ.get("PFB_PARITY_REPORT")  # optional: one JSON line of measured errors per check
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF = [torch.float16, torch.bfloat16]
G = 64  # guard elements before and after every output (keeps 16-byte alignment)


def _report(**kw):
    if not REPORT:
        return
    try:
        os.makedirs(os.path.dirname(REPORT), exist_ok=True)
        with open(REPORT, "a") as f:
            f.write(json.dumps(kw) + "\n")
    except OSError:
        pass


def _seed(*parts):
    return zlib.crc32("/".join(str(p) for p in parts).encode())


def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV) * scale


def _lib():
    from ptlflow_b200 import _lib

    return _lib


def _call(fn, *args, what=""):
    L = _lib()
    L.check(fn(*args), what)


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _guarded(n, dtype, fill=R.SENTINEL):
    """(base, view of n elements) with G sentinel guard elements on either side."""
    base = torch.full((n + 2 * G,), fill, dtype=dtype, device=DEV)
    return base, base[G:G + n]


def _assert_guards(base, what):
    s = torch.full((G,), R.SENTINEL, dtype=base.dtype, device=DEV)
    assert torch.equal(base[:G], s) and torch.equal(base[-G:], s), f"{what}: guard elements written"


def _short(dt):
    return str(dt)[6:]


def _coords(Q, H, W, seed, sigma=3.0):
    """[Q, 2] float32 around an H x W map, with the edge cases listed in the module docstring."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = torch.stack([torch.rand(Q, generator=g, device=DEV) * W, torch.rand(Q, generator=g, device=DEV) * H], 1)
    c = c + sigma * torch.randn(Q, 2, generator=g, device=DEV)
    special = [(3.0, 2.0), (W - 1.0, H / 2), (-1e-7, 1.0), (-40.0, 2.0), (math.nan, 1.0), (1.0, math.inf), (-math.inf, 0.0),
               (W / 2, -1e-7), (W - 1.0, H - 1.0), (W - 0.5, 1.5), (W + 3.5, H - 0.25)]
    for l in range(4):
        t = 1e7 * 2.0 ** l
        below = float(torch.nextafter(torch.tensor(t, dtype=torch.float32), torch.tensor(0.0)))
        special += [(below, 1.0), (t, 1.0), (-t, 1.0), (1.0, -below)]
    special += [(k + 4.25, 2.5) for k in range(8)]  # window origin at tile column k
    special += [(8.0 * (W // 8) + k - 4 + 0.5, H - 2.0) for k in range(8)]  # ... and near the right edge
    assert Q >= len(special)
    c[:len(special)] = torch.tensor(special, dtype=torch.float32, device=DEV)
    return c.float().contiguous()


# =====================================================================================================================
# volume
# =====================================================================================================================
def vcase(name, B, H, W, C, L, target=None, scale=None, wgmma=True, simt=True, tiled=True):
    return dict(name=name, B=B, H=H, W=W, C=C, L=L, target=target, scale=scale, wgmma=wgmma, simt=simt, tiled=tiled)


VOLUME_CASES = [
    vcase("c64_w24_odd_h", 2, 13, 24, 64, 4),             # 2 B stages, TMA store; N = 312
    vcase("c64_grid_5x7", 3, 5, 7, 64, 1),                # smaller than one 8 x 16 patch
    vcase("c128_w21", 1, 11, 21, 128, 4),                 # direct stores (W % 8 != 0): vec0 .. vec3 all off
    vcase("c128_w16_l2", 2, 3, 16, 128, 2),               # TMA store; vec1 (W1 = 8) on
    vcase("c192_w40", 2, 9, 40, 192, 3),                  # 1 B stage, TMA store
    vcase("c192_w36", 1, 17, 36, 192, 4),                 # 1 B stage, direct stores, vec2 (W2 = 9) off
    vcase("c256_w32", 1, 15, 32, 256, 4),                 # never a TMA store; vec0 .. vec3 on
    vcase("c256_w19_n247", 2, 13, 19, 256, 2),
    vcase("grid_55x128_one_group", 5, 55, 128, 64, 4, simt=False, tiled=False),  # groups = 1: a CTA walks every patch
    # a target grid of its own (SEA-RAFT's per-level volumes; FlowFormer's unscaled cost maps)
    vcase("ex_sea_raft", 2, 12, 20, 128, 1, target=(6, 10)),
    vcase("ex_flowformer_unscaled", 1, 10, 14, 256, 3, target=(13, 24), scale=1.0),
    vcase("ex_c64_l4", 1, 7, 9, 64, 4, target=(23, 41)),
]
VBY = {c["name"]: c for c in VOLUME_CASES}


def _vol_inputs(c, dtype):
    B, H1, W1, C = c["B"], c["H"], c["W"], c["C"]
    H2, W2 = c["target"] or (H1, W1)
    sd = _seed(c["name"])
    f1 = _randn((B, H1, W1, C), sd).to(dtype)
    f2 = _randn((B, H2, W2, C), sd + 1).to(dtype)
    scale = c["scale"] if c["scale"] is not None else C ** -0.5
    return f1, f2, H2, W2, scale


def run_volume(c, dtype, impl):
    """Dense pyramid (impl 1 or 2) of case c against the re-rounded bound.  Returns max(err / bound)."""
    lib = _lib().load()
    B, H1, W1, C, L = c["B"], c["H"], c["W"], c["C"], c["L"]
    f1, f2, H2, W2, scale = _vol_inputs(c, dtype)
    Q = B * H1 * W1
    bases, levels = [], []
    for l in range(L):
        base, v = _guarded(Q * (H2 >> l) * (W2 >> l), dtype)
        bases.append(base)
        levels.append(v.view(Q, H2 >> l, W2 >> l))
    L_ = _lib()
    _call(lib.pfb_corr_volume_build_ex, f1.data_ptr(), f2.data_ptr(), L_.ptr_array(levels), B, H1, W1, H2, W2, C, L, scale,
          L_.dtype_code(dtype), impl, _stream(), what="corr_volume_build_ex")
    torch.cuda.synchronize()
    what = f"volume {c['name']} {dtype} impl={impl}"
    ref0, S = R.volume(f1.double(), f2.double(), scale)
    worst = 0.0
    ref, bound = ref0, R.volume_bound(ref0, S, C, scale, dtype)
    del S
    for l in range(L):
        if l:
            ref, bound = R.pool_rerounded(ref, bound, dtype)
        worst = max(worst, R.assert_within(levels[l], ref, bound, f"{what} level {l}"))
        _assert_guards(bases[l], f"{what} level {l}")
    return worst


def _promised_zero(h, w, l):
    """[tiles_y * tiles_x * 32] bool: pad elements the tiled volume kernel writes as zero.  Level 0 leaves through a TMA box
    of whole tiles whose out-of-map targets were zero-filled; levels 1-3 zero the pad columns of the row chunks (8, 4, 2
    columns) they store, in the map's rows."""
    ty, tx = R.t84_shape(h, w)
    y = torch.arange(ty * 4, device=DEV).view(-1, 1).expand(ty * 4, tx * 8)
    x = torch.arange(tx * 8, device=DEV).view(1, -1).expand(ty * 4, tx * 8)
    if l == 0:
        m = (y >= h) | (x >= w)
    else:
        chunk = 16 >> l
        m = (y < h) & (x >= w) & (x < (w + chunk - 1) // chunk * chunk)
    off = ((y >> 2) * tx + (x >> 3)) * 32 + (y & 3) * 8 + (x & 7)
    out = torch.zeros(ty * tx * 32, dtype=torch.bool, device=DEV)
    out[off[m]] = True
    return out


def run_tiled_volume(c, dtype):
    lib = _lib().load()
    L_ = _lib()
    B, H1, W1, C, L = c["B"], c["H"], c["W"], c["C"], c["L"]
    f1, f2, H2, W2, scale = _vol_inputs(c, dtype)
    Q = B * H1 * W1
    bases, levels = [], []
    for l in range(L):
        n = lib.pfb_corr_level_bytes_tiled(B, H1, W1, H2, W2, l) // 2
        base, v = _guarded(n, dtype)
        bases.append(base)
        levels.append(v.view(Q, -1))
    _call(lib.pfb_corr_volume_build_tiled, f1.data_ptr(), f2.data_ptr(), L_.ptr_array(levels), B, H1, W1, H2, W2, C, L, scale,
          L_.dtype_code(dtype), _stream(), what="corr_volume_build_tiled")
    torch.cuda.synchronize()
    what = f"tiled volume {c['name']} {dtype}"
    ref0, S = R.volume(f1.double(), f2.double(), scale)
    worst = 0.0
    for l, (ref, bound) in enumerate(R.pyramid_once(ref0, S, C, scale, dtype, L)):
        h, w = H2 >> l, W2 >> l
        worst = max(worst, R.assert_within(R.t84_read(levels[l], h, w), ref, bound, f"{what} level {l}"))
        z = levels[l][:, _promised_zero(h, w, l)]
        assert bool((z == 0).all()), f"{what} level {l}: pad not zero"
        _assert_guards(bases[l], f"{what} level {l}")
    return worst


def _vol_variants(c):
    v = []
    if c["wgmma"]:
        v += [(dt, 2) for dt in HALF]
    if c["simt"]:
        v += [(dt, 1) for dt in HALF + [torch.float32]]
    return v


VOL_PARAMS = [pytest.param(c["name"], dt, impl, id=f"{c['name']}-{_short(dt)}-impl{impl}") for c in VOLUME_CASES for dt, impl in _vol_variants(c)]


@pytest.mark.parametrize("name,dtype,impl", VOL_PARAMS)
def test_volume_conformance(name, dtype, impl):
    worst = run_volume(VBY[name], dtype, impl)
    _report(test="corr_volume", case=name, dtype=str(dtype), impl=impl, max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", HALF, ids=["float16", "bfloat16"])
@pytest.mark.parametrize("name", [c["name"] for c in VOLUME_CASES if c["tiled"]])
def test_tiled_volume_conformance(name, dtype):
    worst = run_tiled_volume(VBY[name], dtype)
    _report(test="corr_volume_tiled", case=name, dtype=str(dtype), max_err_over_bound=worst)


def run_volume_sweep_direct_stores():
    """The wgmma cases at C <= 192 (test_volume_direct_stores runs this with the level-0 TMA store switched off)."""
    n = 0
    for c in VOLUME_CASES:
        if c["wgmma"] and c["C"] <= 192:
            for dt in HALF:
                run_volume(c, dt, 2)
                n += 1
    print("cases", n)


def test_volume_direct_stores(tmp_path):
    """PFB_VOLUME_TMA_STORE=0 (read once per process): level 0 leaves through the direct vector / scalar stores at every C."""
    env = dict(os.environ, PFB_VOLUME_TMA_STORE="0")
    env.pop("PFB_PARITY_REPORT", None)
    code = "import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; import test_gpu_corr_conformance as T; T.run_volume_sweep_direct_stores()"
    r = subprocess.run([sys.executable, "-c", code, ROOT, os.path.join(ROOT, "tests")], env=env, cwd=str(tmp_path),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert "cases 18" in r.stdout, r.stdout[-400:]


# =====================================================================================================================
# lookup from stored levels
# =====================================================================================================================
LOOKUP_CASES = [
    dict(name="r4_fast", B=1, H=11, W=21, r=4, L=4, nchw=False),
    dict(name="r3_fast", B=2, H=9, W=16, r=3, L=3, nchw=False),
    dict(name="generic_nchw_r4", B=1, H=11, W=21, r=4, L=4, nchw=True),
    dict(name="generic_r5", B=1, H=10, W=19, r=5, L=2, nchw=False),
    dict(name="level_hw_fast", B=1, H=8, W=12, r=4, L=3, nchw=False, level_hw=[(9, 14), (7, 11), (3, 5)]),
    dict(name="level_hw_nchw", B=2, H=6, W=10, r=4, L=2, nchw=True, level_hw=[(13, 24), (4, 7)]),
]
LBY = {c["name"]: c for c in LOOKUP_CASES}


@pytest.mark.parametrize("dtype", HALF + [torch.float32], ids=["float16", "bfloat16", "float32"])
@pytest.mark.parametrize("name", list(LBY))
def test_lookup_conformance(name, dtype):
    c = LBY[name]
    lib, L_ = _lib().load(), _lib()
    B, H, W, r, L, nchw = c["B"], c["H"], c["W"], c["r"], c["L"], c["nchw"]
    Q, K = B * H * W, 2 * r + 1
    sd = _seed(name)
    hw = c.get("level_hw") or [(H >> l, W >> l) for l in range(L)]
    levels = [_randn((Q, h, w), sd + l).to(dtype) for l, (h, w) in enumerate(hw)]
    coords = _coords(Q, hw[0][0], hw[0][1], sd + 9).view(B, H, W, 2)
    planes = L * K * K
    stride = planes if nchw else (planes + 7) // 8 * 8 + 8
    base, flat = _guarded(B * H * W * stride, dtype)
    args = (coords.data_ptr(), flat.data_ptr(), B, H, W, L, r, L_.dtype_code(dtype), L_.dtype_code(dtype), int(nchw), stride, _stream())
    if "level_hw" in c:
        lh = (L_.C.c_int * L)(*[h for h, _ in hw])
        lw = (L_.C.c_int * L)(*[w for _, w in hw])
        _call(lib.pfb_corr_lookup_ex, L_.ptr_array(levels), lh, lw, *args, what="corr_lookup_ex")
    else:
        _call(lib.pfb_corr_lookup, L_.ptr_array(levels), *args, what="corr_lookup")
    torch.cuda.synchronize()
    ref, bound = R.lookup([v.double() for v in levels], coords.view(-1, 2), r, dtype)
    what = f"lookup {name} {dtype}"
    if nchw:
        got = flat.view(B, planes, H, W).permute(0, 2, 3, 1).reshape(Q, planes)
    else:
        rows = flat.view(Q, stride)
        got = rows[:, :planes]
        assert bool((rows[:, planes:] == 0).all()), f"{what}: pad columns not zero"
    worst = R.assert_within(got, ref, bound, what)
    _assert_guards(base, what)
    _report(test="corr_lookup", case=name, dtype=str(dtype), max_err_over_bound=worst)


TILED_RL = [(4, 1), (4, 2), (4, 3), (4, 4), (3, 3), (3, 4)]


def _tiled_lookup(levels_t, coords, B, H, W, H2, W2, r, dtype, stride):
    lib, L_ = _lib().load(), _lib()
    base, flat = _guarded(B * H * W * stride, dtype)
    _call(lib.pfb_corr_lookup_tiled, L_.ptr_array(levels_t), coords.data_ptr(), flat.data_ptr(), B, H, W, H2, W2, len(levels_t), r,
          L_.dtype_code(dtype), stride, _stream(), what="corr_lookup_tiled")
    torch.cuda.synchronize()
    return base, flat


@pytest.mark.parametrize("dtype", HALF, ids=["float16", "bfloat16"])
@pytest.mark.parametrize("targets", [(11, 21), (12, 32)], ids=["t11x21", "t12x32"])
@pytest.mark.parametrize("r,L", TILED_RL)
def test_tiled_lookup_conformance(r, L, targets, dtype):
    B, H, W = 2, 7, 9
    H2, W2 = targets
    Q, K = B * H * W, 2 * r + 1
    sd = _seed("tiled_lookup", r, L, H2, W2)
    hw = [(H2 >> l, W2 >> l) for l in range(L)]
    dense = [_randn((Q, h, w), sd + l).to(dtype) for l, (h, w) in enumerate(hw)]
    coords = _coords(Q, H2, W2, sd + 9).view(B, H, W, 2)
    planes = L * K * K
    stride = (planes + 7) // 8 * 8 + 8
    what = f"tiled lookup r={r} L={L} {targets} {dtype}"
    base, flat = _tiled_lookup([R.t84_write(v, 1000.0) for v in dense], coords, B, H, W, H2, W2, r, dtype, stride)
    rows = flat.view(Q, stride)
    ref, bound = R.lookup([v.double() for v in dense], coords.view(-1, 2), r, dtype)
    worst = R.assert_within(rows[:, :planes], ref, bound, what)
    assert bool((rows[:, planes:] == 0).all()), f"{what}: pad columns not zero"
    _assert_guards(base, what)
    # pad rows / columns poisoned with NaN instead of 1000: the same bits
    _, flat2 = _tiled_lookup([R.t84_write(v, math.nan) for v in dense], coords, B, H, W, H2, W2, r, dtype, stride)
    assert torch.equal(R.bits(flat2), R.bits(flat)), f"{what}: the result depends on the pad"
    _report(test="corr_lookup_tiled", case=f"r{r}_L{L}_{H2}x{W2}", dtype=str(dtype), max_err_over_bound=worst)


@pytest.mark.parametrize("dtype", HALF + [torch.float32], ids=["float16", "bfloat16", "float32"])
def test_avg_pool2x2_odd_sizes(dtype):
    lib, L_ = _lib().load(), _lib()
    N, H, W, C = 3, 7, 9, 24
    x = _randn((N, H, W, C), _seed("pool")).to(dtype)
    base, flat = _guarded(N * (H // 2) * (W // 2) * C, dtype)
    _call(lib.pfb_avg_pool2x2_nhwc, x.data_ptr(), flat.data_ptr(), N, H, W, C, L_.dtype_code(dtype), _stream(), what="avg_pool2x2")
    torch.cuda.synchronize()
    worst = R.assert_within(flat.view(N, H // 2, W // 2, C), *R.avg_pool2x2(x.double(), dtype), what=f"avg_pool2x2 {dtype}")
    _assert_guards(base, f"avg_pool2x2 {dtype}")
    _report(test="avg_pool2x2", case="7x9", dtype=str(dtype), max_err_over_bound=worst)


# =====================================================================================================================
# on the fly
# =====================================================================================================================
def ocase(name, B, H, W, C, L, sigma, creal=None, mag=1.0, coords=None):
    return dict(name=name, B=B, H=H, W=W, C=C, L=L, sigma=sigma, creal=creal or C, mag=mag, coords=coords)


OTF_CASES = [
    ocase("c64_smooth", 2, 20, 40, 64, 4, 0.0),          # n_items 72 > 2 x grid 18
    ocase("c128_rough", 1, 24, 48, 128, 4, 4.0),
    ocase("c192_very_rough", 1, 30, 40, 192, 3, 12.0),
    ocase("c256", 1, 17, 35, 256, 4, 2.0),
    ocase("c96_padded_128", 2, 16, 24, 128, 4, 3.0, creal=96),
    ocase("bands_2_to_8", 1, 64, 128, 64, 1, 0.0, coords="bands"),
    # |a.b| above 65504 in f16 with the scaled correlation well inside it (the tensor-core dump once rounded the raw dot:
    # inf for the queries its region served, finite for the flagged ones)
    ocase("f16_dot_overflow", 1, 16, 32, 256, 2, 0.0, mag=20.0, coords="overflow"),
]
OBY = {c["name"]: c for c in OTF_CASES}


def _otf_inputs(c, dtype):
    B, H, W, C, Cr, L = c["B"], c["H"], c["W"], c["C"], c["creal"], c["L"]
    sd = _seed(c["name"])
    f1 = torch.zeros((B, H, W, C), device=DEV)
    f2 = torch.zeros((B, H, W, C), device=DEV)
    f1[..., :Cr] = _randn((B, H, W, Cr), sd, c["mag"])
    f2[..., :Cr] = _randn((B, H, W, Cr), sd + 1, c["mag"])
    if c["coords"] == "overflow":
        f2 = f1.clone()  # the window centre tap of a query on its own pixel: |a|^2 ~ 256 * 400
    f1, f2 = f1.to(dtype), f2.to(dtype)
    from ptlflow_b200 import ops

    pyr = [f2]
    for _ in range(L - 1):
        pyr.append(ops.avg_pool2x2(pyr[-1]))
    ys, xs = torch.meshgrid(torch.arange(H, device=DEV, dtype=torch.float32), torch.arange(W, device=DEV, dtype=torch.float32), indexing="ij")
    grid = torch.stack([xs, ys], -1)[None].repeat(B, 1, 1, 1)
    g = torch.Generator(device=DEV).manual_seed(sd + 2)
    coords = grid + c["sigma"] * torch.randn(grid.shape, generator=g, device=DEV)
    if c["coords"] == "bands":  # tile k: window rows spread over 7 nb - 15 rows, nb = 2 + k % 7
        tiles_x = (W + 15) // 16
        t = (torch.arange(H, device=DEV) // 8).view(-1, 1) * tiles_x + (torch.arange(W, device=DEV) // 16).view(1, -1)
        spread = (7 * (2 + t % 7) - 15).clamp_min(0).float()
        last_row = (torch.arange(H, device=DEV) % 8 == 7).view(-1, 1)
        coords[..., 1] = 4.0 + torch.where(last_row, spread, torch.zeros_like(spread))
        coords[:, H - 8:, :W // 2] = math.nan  # tiles without a live query
        coords[:, H - 8:, W // 2:] = -30.0     # ... and with every window left of and above the map
    elif c["coords"] == "overflow":  # rows 8..15: rough, so that some queries are flagged
        coords[:, 8:] += 9.0 * torch.randn(coords[:, 8:].shape, generator=g, device=DEV)
    else:
        flat = coords.view(-1, 2)
        flat[:16] = _coords(64, H, W, sd + 3)[:16]  # NaN, inf, far-away and edge coordinates
    return f1, pyr, coords.contiguous(), c["creal"] ** -0.5


def run_otf(c, dtype, tensor_cores):
    """Returns (max err / bound, flags or None)."""
    lib, L_ = _lib().load(), _lib()
    B, H, W, C, L = c["B"], c["H"], c["W"], c["C"], c["L"]
    f1, pyr, coords, scale = _otf_inputs(c, dtype)
    Q, planes = B * H * W, L * 81
    stride = (planes + 7) // 8 * 8 + 8
    base, flat = _guarded(Q * stride, dtype)
    dt = L_.dtype_code(dtype)
    flags = None
    if tensor_cores:
        ws = torch.full((lib.pfb_corr_lookup_onthefly_tc_workspace_bytes(B, H, W),), 7, dtype=torch.uint8, device=DEV)
        if c["creal"] == C:
            _call(lib.pfb_corr_lookup_onthefly_tc, f1.data_ptr(), L_.ptr_array(pyr), coords.data_ptr(), flat.data_ptr(), ws.data_ptr(),
                  B, H, W, C, L, 4, dt, stride, _stream(), what="corr_lookup_onthefly_tc")
        else:
            _call(lib.pfb_corr_lookup_onthefly_tc_ex, f1.data_ptr(), L_.ptr_array(pyr), coords.data_ptr(), flat.data_ptr(), ws.data_ptr(),
                  B, H, W, C, L, 4, scale, dt, stride, _stream(), what="corr_lookup_onthefly_tc_ex")
        flags = ws
    else:
        _call(lib.pfb_corr_lookup_onthefly_ex, f1.data_ptr(), L_.ptr_array(pyr), coords.data_ptr(), flat.data_ptr(), B, H, W, C, L, 4,
              scale, dt, dt, 0, stride, _stream(), what="corr_lookup_onthefly_ex")
    torch.cuda.synchronize()
    what = f"on the fly {c['name']} {dtype} {'tensor cores' if tensor_cores else 'simt'}"
    ref, bound = R.onthefly(f1.double(), [p.double() for p in pyr], coords.view(-1, 2), 4, scale, dtype, tensor_cores)
    rows = flat.view(Q, stride)
    worst = R.assert_within(rows[:, :planes], ref, bound, what)
    assert bool((rows[:, planes:] == 0).all()), f"{what}: pad columns not zero"
    _assert_guards(base, what)
    if tensor_cores:
        _, _, _, want = R.otf_plan(coords, H, W, L)
        got = flags.view(B, H, W)
        assert bool(((got == 0) | (got == 1)).all()), f"{what}: flags not 0 / 1"
        assert torch.equal(got.bool(), want), f"{what}: {int((got.bool() != want).sum())} flags differ from the region rule"
    return worst


OTF_PARAMS = ([pytest.param(c["name"], dt, tc, id=f"{c['name']}-{_short(dt)}-{'tc' if tc else 'simt'}")
               for c in OTF_CASES for dt in HALF for tc in (True, False)]
              + [pytest.param(c["name"], torch.float32, False, id=f"{c['name']}-float32-simt") for c in OTF_CASES])


@pytest.mark.parametrize("name,dtype,tensor_cores", OTF_PARAMS)
def test_onthefly_conformance(name, dtype, tensor_cores):
    worst = run_otf(OBY[name], dtype, tensor_cores)
    _report(test="corr_onthefly", case=name, dtype=str(dtype), impl="tc" if tensor_cores else "simt", max_err_over_bound=worst)


def test_onthefly_plan_coverage():
    """Across the sweep the region rule reaches every band count a live tile can have (2 .. 8: one band of 8 rows never
    holds a 10-row window) and tiles without live queries (0), tiles that mix flagged and unflagged queries, negative
    anchors, and more than two work items per CTA."""
    nbs, mixed, negative, wrapped = set(), False, False, False
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    for c in OTF_CASES:
        _, _, coords, _ = _otf_inputs(c, torch.float16)
        nb, bx, by, flags = R.otf_plan(coords, c["H"], c["W"], c["L"])
        nbs |= set(nb.tolist())
        negative |= bool(((bx < 0) | (by < 0)).any())
        B, H, W = c["B"], c["H"], c["W"]
        ty, tx = (H + 7) // 8, (W + 15) // 16
        f = torch.zeros((B, ty * 8, tx * 16), dtype=torch.float32, device=DEV)
        v = torch.zeros_like(f)
        f[:, :H, :W], v[:, :H, :W] = flags.float(), 1.0
        per = f.view(B, ty, 8, tx, 16).sum((2, 4))
        cnt = v.view(B, ty, 8, tx, 16).sum((2, 4))
        mixed |= bool(((per > 0) & (per < cnt)).any())
        n_tiles = B * ty * tx
        wrapped |= n_tiles * c["L"] > 2 * min(sms, n_tiles)
    assert {0, 2, 3, 4, 5, 6, 7, 8} <= nbs, sorted(nbs)
    assert mixed and negative and wrapped


def run_otf_trace_sweep(plan_path):
    """Every on-the-fly case once on the tensor cores (f16), and otf_plan's band counts per case (test_onthefly_trace)."""
    plans = []
    for c in OTF_CASES:
        run_otf(c, torch.float16, True)
        _, _, coords, _ = _otf_inputs(c, torch.float16)
        plans.append(R.otf_plan(coords, c["H"], c["W"], c["L"])[0].tolist())
    with open(plan_path, "w") as f:
        json.dump(plans, f)


def test_onthefly_trace(tmp_path):
    """Stamp slot 2 of every CTA under PFB_OTF_TRACE is the band count of the CTA's second work item."""
    trace, plan = tmp_path / "otf_trace.jsonl", tmp_path / "plans.json"
    env = dict(os.environ, PFB_OTF_TRACE=str(trace))
    env.pop("PFB_PARITY_REPORT", None)
    code = ("import sys; sys.path[:0] = [sys.argv[1], sys.argv[2]]; import test_gpu_corr_conformance as T; "
            "T.run_otf_trace_sweep(sys.argv[3])")
    r = subprocess.run([sys.executable, "-c", code, ROOT, os.path.join(ROOT, "tests"), str(plan)], env=env, cwd=str(tmp_path),
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    lines = [json.loads(x) for x in trace.read_text().splitlines() if x.strip()]
    plans = json.loads(plan.read_text())
    assert len(lines) == len(plans) == len(OTF_CASES)
    checked = 0
    for c, t, nb in zip(OTF_CASES, lines, plans):
        grid = t["grid"]
        assert (t["H"], t["W"], t["kchunks"]) == (c["H"], c["W"], c["C"] // 64)
        stamps = t["stamps"]
        for cta in range(grid):
            item = cta + grid
            if item < len(nb):
                assert stamps[cta * 64 + 2] == nb[item], (c["name"], cta, stamps[cta * 64 + 2], nb[item])
                checked += 1
    assert checked > 0


# =====================================================================================================================
# calls that are refused without a launch
# =====================================================================================================================
def _refused(fn, *args, match=None):
    lib = _lib().load()
    torch.cuda.synchronize()
    n0 = lib.pfb_launch_count(-1)
    rc = fn(*args)
    torch.cuda.synchronize()
    assert rc != 0
    if match:
        assert match in lib.pfb_last_error().decode(), lib.pfb_last_error()
    assert lib.pfb_launch_count(-1) == n0


def _tiled_refusal_args():
    B, H, W, H2, W2 = 1, 4, 8, 8, 16
    levels = [torch.zeros((B * H * W, 32 * math.prod(R.t84_shape(H2 >> l, W2 >> l))), dtype=torch.float16, device=DEV) for l in range(2)]
    coords = torch.zeros((B, H, W, 2), device=DEV)
    out = torch.zeros(B * H * W * 104 + 8, dtype=torch.float16, device=DEV)
    return levels, coords, out, (B, H, W, H2, W2)


def test_tiled_lookup_refusals():
    lib, L_ = _lib().load(), _lib()
    levels, coords, out, shape = _tiled_refusal_args()
    dt = L_.dtype_code(torch.float16)
    _refused(lib.pfb_corr_lookup_tiled, L_.ptr_array(levels[:1]), coords.data_ptr(), out.data_ptr(), *shape, 1, 4, dt, 84,
             _stream(), match="multiple of 8")
    _refused(lib.pfb_corr_lookup_tiled, L_.ptr_array(levels[:1]), coords.data_ptr(), out.data_ptr() + 2, *shape, 1, 4, dt, 88,
             _stream(), match="16-byte aligned")


def test_tiled_lookup_uninstantiated_radius_counts_no_launch():
    """R = 3 with two levels has no kernel: refused, and (it once was not) without counting a launch."""
    lib, L_ = _lib().load(), _lib()
    levels, coords, out, shape = _tiled_refusal_args()
    _refused(lib.pfb_corr_lookup_tiled, L_.ptr_array(levels), coords.data_ptr(), out.data_ptr(), *shape, 2, 3,
             L_.dtype_code(torch.float16), 104, _stream(), match="not instantiated")


def test_tiled_volume_refusals():
    from ptlflow_b200 import ops

    lib = _lib().load()
    for dtype, C in ((torch.float16, 96), (torch.float32, 64)):
        f = torch.zeros((1, 8, 16, C), dtype=dtype, device=DEV)
        torch.cuda.synchronize()
        n0 = lib.pfb_launch_count(-1)
        with pytest.raises(RuntimeError, match="corr_volume_build_tiled"):
            ops.corr_volume_build_tiled(f, f, 2)
        torch.cuda.synchronize()
        assert lib.pfb_launch_count(-1) == n0


def test_onthefly_tc_refusals():
    lib, L_ = _lib().load(), _lib()
    B, H, W = 1, 8, 16
    ws = torch.zeros(B * H * W, dtype=torch.uint8, device=DEV)
    coords = torch.zeros((B, H, W, 2), device=DEV)
    out = torch.zeros(B * H * W * 88, dtype=torch.float16, device=DEV)
    for C, r in ((64, 3), (96, 4)):
        f = torch.zeros((B, H, W, C), dtype=torch.float16, device=DEV)
        _refused(lib.pfb_corr_lookup_onthefly_tc, f.data_ptr(), L_.ptr_array([f]), coords.data_ptr(), out.data_ptr(), ws.data_ptr(),
                 B, H, W, C, 1, r, L_.dtype_code(torch.float16), 88, _stream(), match="radius 4")
