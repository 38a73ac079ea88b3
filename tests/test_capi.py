"""CPU: the C-ABI library builds for sm_90a, loads without a GPU, exports every symbol the header
declares, and rejects bad arguments with an error message before touching the device."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "ptlflow_b200.h")


@pytest.fixture(scope="module")
def lib():
    from ptlflow_b200.csrc import build as B
    from ptlflow_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        B.build()
    return _lib.load()


def declared_symbols():
    text = open(HEADER).read()
    return sorted(set(re.findall(r"PFB_API[^;(]*?\b(pfb_\w+)\s*\(", text)))


def test_header_symbols_are_exported_and_bound(lib):
    from ptlflow_b200 import _lib

    names = declared_symbols()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ptlflow_b200.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in ptlflow_b200/_lib.py"
    assert sorted(_lib.SIGNATURES) == names


def test_kernel_class_names_match_the_header():
    """One name per profiler class: a class added to the header without a name here would drop out of every split."""
    from ptlflow_b200 import _lib

    declared = int(re.search(r"#define\s+PFB_KERNEL_CLASSES\s+(\d+)", open(HEADER).read()).group(1))
    assert len(_lib.KERNEL_CLASS_NAMES) == _lib.KERNEL_CLASSES == declared
    assert len(set(_lib.KERNEL_CLASS_NAMES)) == declared


def test_version_and_error_channel(lib):
    assert lib.pfb_version() >= 100
    rc = lib.pfb_corr_lookup(None, None, None, 1, 8, 8, 4, 4, 0, 0, 0, 324, None)
    assert rc == -1
    assert b"null pointer" in lib.pfb_last_error()


def test_argument_validation_without_device(lib):
    from ptlflow_b200 import _lib

    dummy = (C.c_void_p * 8)(*([1] * 8))
    pp = C.cast(dummy, C.POINTER(C.c_void_p))
    # 4 levels on an 4x4 grid: level 3 would be empty
    assert lib.pfb_corr_volume_build(1, 1, pp, 1, 4, 4, 64, 4, 0, 1, None) == -1
    assert b"too small" in lib.pfb_last_error()
    # bad dtype / radius
    assert lib.pfb_corr_lookup(pp, 1, 1, 1, 8, 8, 1, 4, 7, 0, 0, 81, None) == -1
    assert lib.pfb_corr_lookup(pp, 1, 1, 1, 8, 8, 1, 99, 0, 0, 0, 81, None) == -1
    # out_stride smaller than the number of lookup planes
    assert lib.pfb_corr_lookup(pp, 1, 1, 1, 8, 8, 1, 4, 0, 0, 0, 80, None) == -1
    # on-the-fly needs C % 8 == 0
    assert lib.pfb_corr_lookup_onthefly(1, pp, 1, 1, 1, 8, 8, 30, 1, 4, 0, 0, 1, 0, None) == -1
    # conv: even kernel
    p = _lib.ConvParams()
    p.nsrc, p.B, p.H, p.W, p.KH, p.KW, p.Cout, p.Cout_pad = 1, 1, 4, 4, 2, 3, 8, 8
    p.src[0] = _lib.ConvSrc(1, 8, 8, 0, 0)
    p.weight, p.out = 1, 1
    assert lib.pfb_conv2d(C.byref(p), None) == -1
    assert b"odd" in lib.pfb_last_error()


def test_workspace_plan_is_host_only(lib):
    from ptlflow_b200 import _lib

    cfg = _lib.RaftCfg(0, _lib.F16, 8, 55, 128, 256, 4, 4, 128, 128, 12, 0, 436, 1024, 2, 0, 0)
    n = lib.pfb_raft_workspace_bytes(C.byref(cfg))
    P = 8 * 55 * 128
    assert n >= P * (384 + 256 + 256 + 128 + 128 + 128 + 128 + 256 + 256 + 576) * 2
    assert n < 2 * P * 2600 * 2
    small = _lib.RaftCfg(1, _lib.F32, 1, 16, 32, 128, 4, 3, 96, 64, 4, 0, 128, 256, 0, 0, 0)
    assert lib.pfb_raft_workspace_bytes(C.byref(small)) > 0
    bad = _lib.RaftCfg(0, _lib.F32, 1, 16, 32, 128, 4, 3, 96, 64, 4, 0, 128, 256, 0, 0, 0)  # raft needs hidden 128
    assert lib.pfb_raft_workspace_bytes(C.byref(bad)) == 0


def test_missing_library_is_loud(monkeypatch, tmp_path):
    from ptlflow_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.LibraryMissing):
        _lib.load()


def test_struct_fields_match_the_header():
    """Field names and order of every struct in include/ptlflow_b200.h equal the ctypes mirrors in ptlflow_b200/_lib.py
    (a field added on one side only would shift everything behind it silently)."""
    import re

    from ptlflow_b200 import _lib

    text = open(os.path.join(ROOT, "include", "ptlflow_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)  # comments out
    mirrors = {"pfb_conv_src": _lib.ConvSrc, "pfb_conv_params": _lib.ConvParams, "pfb_layer": _lib.Layer, "pfb_raft_cfg": _lib.RaftCfg,
               "pfb_raft_weights": _lib.RaftWeights, "pfb_raft_buffers": _lib.RaftBuffers}
    found = 0
    for body, name in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", text, flags=re.S):
        if name not in mirrors:
            continue
        found += 1
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            # "int a, b, c" / "const void* weight" / "pfb_conv_src src[PFB_MAX_SRC]" / "void* const* pyramid"
            first, *rest = [d.strip() for d in decl.split(",")]
            names = [re.sub(r"\[.*\]", "", first.split()[-1]).lstrip("*")] + [re.sub(r"\[.*\]", "", r).lstrip("*").strip() for r in rest]
            fields += names
        mirror = [f[0] for f in mirrors[name]._fields_]
        assert fields == mirror, f"{name}: header {fields} != ctypes {mirror}"
    assert found == len(mirrors)
