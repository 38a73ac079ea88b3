"""CPU: which of RAFT's refinement-loop convolutions the wgmma path runs as 256-pixel work items (conv_wide_kernel in
csrc/conv_umma.cu) at the benchmark's grid, per storage type, and that every plan fits the 227 KB of shared memory a block
may use.  pfb_conv2d_umma_plan is the host-only planner that pfb_conv2d's launch calls, so no device is needed."""
import ctypes as C

import pytest
import torch

B, H, W = 8, 55, 128  # 1024x436 frames at 1/8 resolution, 8 pairs (bench.py's workload)
SMEM_LIMIT = 227 * 1024
FAKE = 1 << 20  # an aligned address: the planner only checks alignment

RELU, GRU_ZR, GRU_Q, RELU_APPEND_FLOW, LINEAR_F32, LINEAR = 1, 2, 3, 5, 7, 0
# (name, KH, KW, Cin, Cout, epilogue) of RAFT's basic update block as the loop launches it (csrc/refine.cu): convc1 reads
# the 324-channel lookup, the GRU gates take [h | motion features] with the context part as a per-pixel addend, conv
# appends the flow to its 126 channels, flow2T is the flow head's 1x1 tap-product layer.
LAYERS = [
    ("convc1", 1, 1, 324, 256, RELU),
    ("convc2", 3, 3, 256, 192, RELU),
    ("convf2", 3, 3, 128, 64, RELU),
    ("conv", 3, 3, 256, 126, RELU_APPEND_FLOW),
    ("gru_zr_1x5", 1, 5, 256, 256, GRU_ZR),
    ("gru_q_1x5", 1, 5, 256, 128, GRU_Q),
    ("gru_zr_5x1", 5, 1, 256, 256, GRU_ZR),
    ("gru_q_5x1", 5, 1, 256, 128, GRU_Q),
    ("flow1", 3, 3, 128, 256, RELU),
    ("flow2T", 1, 1, 256, 32, LINEAR_F32),
    ("mask1", 3, 3, 128, 256, RELU),
    ("mask2", 1, 1, 256, 576, LINEAR),
]
WIDE = {"convc2", "conv", "flow1", "mask1"}


@pytest.fixture(scope="module")
def lib():
    import os

    from ptlflow_b200 import _lib
    from ptlflow_b200.csrc import build

    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib


def plan(_lib, KH, KW, Cin, Cout, epi, dtype, b=B, h=H, w=W):
    p = _lib.ConvParams()
    p.src[0] = _lib.ConvSrc(FAKE, Cin, (Cin + 7) // 8 * 8, 0, 0)
    p.nsrc = 1
    p.B, p.H, p.W, p.KH, p.KW = b, h, w, KH, KW
    cout_pad_k = (Cout + 31) // 32 * 32
    p.Cout, p.Cout_pad, p.Cout_pad_k = Cout, cout_pad_k, cout_pad_k
    p.Cin_pad = (Cin + 63) // 64 * 64
    p.weight, p.weight_k, p.bias, p.out, p.flow = FAKE, FAKE, FAKE, FAKE, FAKE
    p.epilogue = epi
    p.out_stride = 32 if epi == LINEAR_F32 else cout_pad_k
    if epi in (GRU_ZR, GRU_Q):
        p.hidden = 128
        p.aux_h = p.aux_z = p.addend = FAKE
        p.addend_stride = cout_pad_k
        p.out_stride = 128
    p.dtype = {torch.float16: 1, torch.bfloat16: 2}[dtype]
    pix, nt, smem = C.c_int(), C.c_int(), C.c_size_t()
    assert _lib.load().pfb_conv2d_umma_plan(C.byref(p), C.byref(pix), C.byref(nt), C.byref(smem)) == 0
    return pix.value, nt.value, smem.value


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["float16", "bfloat16"])
def test_raft_loop_routing(lib, dtype):
    routed = {}
    for name, KH, KW, Cin, Cout, epi in LAYERS:
        pix, nt, smem = plan(lib, KH, KW, Cin, Cout, epi, dtype)
        assert pix in (128, 256), (name, pix)  # every layer runs on the wgmma path
        assert 0 < smem <= SMEM_LIMIT, (name, smem)
        routed[name] = pix == 256
    assert {n for n, r in routed.items() if r} == WIDE
    # the N tiles the 256-pixel items take: convc2's 192 channels as two tiles of 96, the others 128
    assert plan(lib, 3, 3, 256, 192, RELU, dtype)[1] == 96
    assert plan(lib, 3, 3, 128, 256, RELU, dtype)[1] == 128


def test_grids_the_wide_items_waste_stay_on_128_pixels(lib):
    # 128-pixel rows on a 21-pixel-wide grid would compute 6x the pixels; 100 and 200 waste 28 %
    assert plan(lib, 3, 3, 256, 126, RELU_APPEND_FLOW, torch.float16, 2, 11, 21)[0] == 128
    assert plan(lib, 3, 3, 256, 126, RELU_APPEND_FLOW, torch.float16, 2, 11, 100)[0] == 256
    assert plan(lib, 3, 3, 256, 192, RELU, torch.float16, 2, 5, 200)[0] == 256
    assert plan(lib, 3, 3, 256, 192, RELU, torch.float16, 2, 5, 130)[0] == 128


def test_fp32_is_declined(lib):
    p = lib.ConvParams()
    p.dtype = 0
    pix, nt, smem = C.c_int(7), C.c_int(7), C.c_size_t(7)
    assert lib.load().pfb_conv2d_umma_plan(C.byref(p), C.byref(pix), C.byref(nt), C.byref(smem)) == 0
    assert (pix.value, nt.value, smem.value) == (0, 0, 0)
