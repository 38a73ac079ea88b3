"""RaftEngine: packed weights + workspaces + one C call for the whole refinement loop.

This is the host-side glue between the kept ``RAFT.forward`` structure
(ptlflow/models/raft/raft.py:125-194) and ``pfb_raft_refine``.  It owns nothing numerical:
packing, buffers, pointer structs, CUDA-graph capture.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import warnings
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib, ops
from ._lib import check, dtype_code, load, ptr_array, stream_ptr
from .ops import ConvWeights


_TILED = bool(int(os.environ.get("PFB_VOLUME_TILED", "1")))


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return t.data_ptr() if t is not None else None


def _taps(w: torch.Tensor) -> ConvWeights:
    """A 3x3 -> 2 convolution as a 1x1 layer producing the 9 x 2 per-tap products (row = tap*2 + o); the gather adds the bias."""
    return ConvWeights(w.detach().permute(2, 3, 0, 1).reshape(18, w.shape[1], 1, 1).contiguous())


def _pack_convf1(conv: torch.nn.Module, dtype: torch.dtype, device: torch.device) -> ops.PackedConv:
    """The motion encoder's 7x7 convolution of the 2-channel fp32 flow (a dedicated kernel).  In f16 / bf16 with 128 outputs it runs
    in tensor-core form (csrc/first_conv.cu): the K-major slot of the layer carries the overlapping-window tiles."""
    pc = ops.PackedConv([conv], dtype, device)
    if dtype != torch.float32 and tuple(conv.weight.shape) == (128, 2, 7, 7):
        pc.weight_k = ops.pack_flow_conv(conv.weight, dtype).to(device)
        pc.Cin_pad, pc.Cout_pad_k = 64, 128
    return pc


class RaftEngine:
    """Built lazily at first forward and rebuilt when the parameters' dtype / device / storage
    change (callers do ``model.eval().cuda().half()`` *after* construction and after
    ``load_state_dict`` -- model_benchmark.py:274-279, infer.py:148-152).  The model keys it on ``signature``.

    The subclasses share this lifecycle and pack their own weights (``_pack``).  Nothing here changes per call: the engine is shared by
    every host thread that runs the model."""

    # C entry points of this engine's loop (the subclasses run their own with the same cfg / buffers)
    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_raft_workspace_bytes", "pfb_raft_refine", "pfb_raft_update_iter"
    upsample = 8  # the convex upsample's factor: its mask has 9 * upsample**2 channels

    def __init__(self, module: torch.nn.Module, variant: int, hidden_dim: int, context_dim: int, corr_levels: int, corr_radius: int,
                 dtype: torch.dtype, device: torch.device, impl: int = 0, **pack_args):
        self.variant, self.hidden_dim, self.context_dim = variant, hidden_dim, context_dim
        self.corr_levels, self.corr_radius = corr_levels, corr_radius
        self.dtype, self.device, self.impl = dtype, device, impl
        self.agg_gamma, self.num_heads = 0.0, 1
        self.agg_score: Optional[torch.Tensor] = None  # craft: the aggregator's feat2score weight (pfb_raft_buffers.agg_score)
        self.pool_min_side = 0  # how build_volume sizes the pyramid's levels (pfb_raft_buffers.pool_min_side; lcv: 2r+1)
        self.signature = None  # what the model built this engine for (RAFT._get_engine)
        self._keep: List[object] = []  # everything the weight structs point into
        self._workspaces: Dict[int, Tuple] = {}
        self.weights = self._pack(module, **pack_args)
        # the pack kernels ran on the constructing thread's stream; other streams / host threads (pipeline slots) may use
        # the packed weights as soon as the engine is published, so finish them first (one-time cost)
        torch.cuda.current_stream(device).synchronize()

    def _layer(self, pc: ops.PackedConv) -> _lib.Layer:
        self._keep.append(pc)
        return pc.layer_struct()

    def _conv(self, conv, srcs: Optional[List[int]]) -> _lib.Layer:
        """``conv`` (anything with a conv's weight / bias) packed for sources of ``srcs`` channels, kept alive."""
        return self._layer(ops.PackedConv([conv], self.dtype, self.device, src_channels=srcs))

    def _pack(self, update_block: torch.nn.Module, attention_module: Optional[torch.nn.Module] = None) -> _lib.RaftWeights:
        """RAFT's BasicUpdateBlock (gma's, ms_raft_p's and ccmr's too) or raft_small's SmallUpdateBlock."""
        dtype, device, variant = self.dtype, self.device, self.variant
        ub = update_block
        enc, gru, fh = ub.encoder, ub.gru, ub.flow_head
        planes = enc.convc1.in_channels  # levels * (2r+1)^2 planes, or flow1d's 2 (2r+1)
        hd, cd = self.hidden_dim, self.context_dim

        def P(srcs, *convs):  # srcs: channel counts of the concatenated inputs, in order (wgmma K-major pack)
            return ops.PackedConv(convs, dtype, device, src_channels=srcs)

        layers: Dict[int, ops.PackedConv] = {}
        layers[_lib.L_CONVF1] = _pack_convf1(enc.convf1, dtype, device)
        if variant != _lib.VARIANT_RAFT_SMALL:
            layers[_lib.L_CONVC1] = P([planes], enc.convc1)
            layers[_lib.L_CONVC2] = P([256], enc.convc2)
            layers[_lib.L_CONVF2] = P([128], enc.convf2)
            layers[_lib.L_CONV] = P([256], enc.conv)  # cat[cor(192), flo(64)] lives in one 256-channel buffer
            # cat[h or r*h, inp, motion (, motion_global)] -- three tensor maps, no concat copy (gma keeps
            # motion | motion_global in one 256-channel buffer, and so does ccmr: the GRU's input beyond [h | inp])
            gsrc = [hd, cd, gru.convz1.in_channels - hd - cd]
            layers[_lib.L_GRU_ZR1] = P(gsrc, gru.convz1, gru.convr1)  # z | r share the input: one GEMM, N = 2*hidden
            layers[_lib.L_GRU_Q1] = P(gsrc, gru.convq1)
            layers[_lib.L_GRU_ZR2] = P(gsrc, gru.convz2, gru.convr2)
            layers[_lib.L_GRU_Q2] = P(gsrc, gru.convq2)
            if dtype != torch.float32:
                # round 2: (a) the context columns of the four GRU convolutions become layers of their own, evaluated once per
                # forward with the bias folded in, and the per-iteration layers lose them (-1/3 of the GRU's K); (b) convc2 |
                # convf2 as one block-diagonal N = 256 layer.  Pure repacking of the same parameters.
                def cols(conv, lo, hi, with_bias):
                    return ConvWeights(conv.weight.detach()[:, lo:hi].contiguous(), conv.bias if with_bias else None)

                def rest(conv):  # [h | inp | motion...] without the inp columns
                    w = conv.weight.detach()
                    return ConvWeights(torch.cat([w[:, :hd], w[:, hd + cd:]], dim=1).contiguous())

                xsrc = [hd, gsrc[2]]
                for ctx_id, x_id, convs in ((_lib.L_CTX_ZR1, _lib.L_GRUX_ZR1, (gru.convz1, gru.convr1)), (_lib.L_CTX_Q1, _lib.L_GRUX_Q1, (gru.convq1,)),
                                            (_lib.L_CTX_ZR2, _lib.L_GRUX_ZR2, (gru.convz2, gru.convr2)), (_lib.L_CTX_Q2, _lib.L_GRUX_Q2, (gru.convq2,))):
                    layers[ctx_id] = P([cd], *[cols(cv, hd, hd + cd, True) for cv in convs])
                    layers[x_id] = P(xsrc, *[rest(cv) for cv in convs])
                wc, wf = enc.convc2.weight.detach(), enc.convf2.weight.detach()
                if tuple(wc.shape[2:]) == tuple(wf.shape[2:]) and wc.shape[0] + wf.shape[0] == 256:
                    bd = torch.zeros((256, wc.shape[1] + wf.shape[1]) + tuple(wc.shape[2:]), dtype=wc.dtype, device=wc.device)
                    bd[: wc.shape[0], : wc.shape[1]] = wc
                    bd[wc.shape[0]:, wc.shape[1]:] = wf
                    layers[_lib.L_CONVC2F2] = P([wc.shape[1], wf.shape[1]], ConvWeights(bd, torch.cat([enc.convc2.bias.detach(), enc.convf2.bias.detach()])))
            layers[_lib.L_FLOW1] = P([hd], fh.conv1)
            layers[_lib.L_FLOW2] = P([256], fh.conv2)
            if dtype != torch.float32:
                layers[_lib.L_FLOW2T] = P([256], _taps(fh.conv2.weight))
            layers[_lib.L_MASK1] = P([hd], ub.mask[0])
            layers[_lib.L_MASK2] = P([256], ub.mask[2])
        else:  # raft_small: odd channel counts (96 / 82 / 146) -> SIMT kernels only
            layers[_lib.L_CONVC1] = P(None, enc.convc1)
            layers[_lib.L_CONVF2] = P(None, enc.convf2)
            layers[_lib.L_CONV] = P(None, enc.conv)
            layers[_lib.L_GRU_ZR1] = P(None, gru.convz, gru.convr)
            layers[_lib.L_GRU_Q1] = P(None, gru.convq)
            layers[_lib.L_FLOW1] = P(None, fh.conv1)
            layers[_lib.L_FLOW2] = P(None, fh.conv2)
        self.att_q = self.att_k = self.att_pos = None
        if variant == _lib.VARIANT_GMA:
            layers[_lib.L_AGG_V], proj = self._pack_attention(ub.aggregator, attention_module)
            if proj is not None:
                layers[_lib.L_AGG_PROJ] = proj
        self.layers = layers
        w = _lib.RaftWeights()
        for k, v in layers.items():
            w.layers[k] = v.layer_struct()
        return w

    def _pack_attention(self, agg: torch.nn.Module, attention_module: torch.nn.Module):
        """GMA's Aggregate and Attention (gma_utils.py:32-113): sets num_heads, agg_gamma and the per-head q / k / position layers
        of the attention; returns the packed (to_v, project or None) of the per-iteration aggregate."""
        dtype, device = self.dtype, self.device
        self.num_heads = agg.heads
        to_v = ops.PackedConv([agg.to_v], dtype, device, src_channels=[128])
        proj = ops.PackedConv([agg.project], dtype, device, src_channels=[agg.project.weight.shape[1]]) if agg.project is not None else None
        self.agg_gamma = float(agg.gamma.detach().float().cpu().item())

        # one head's q / k block of Attention.to_qk as a 1x1 layer (contiguous head-major outputs for the GEMM)
        wqk = attention_module.to_qk.weight
        c = wqk.shape[0] // 2
        d = c // self.num_heads  # dim_head
        cin = [wqk.shape[1]]
        self.att_q = [ops.PackedConv([ConvWeights(wqk[h * d:(h + 1) * d])], dtype, device, src_channels=cin) for h in range(self.num_heads)]
        self.att_k = [ops.PackedConv([ConvWeights(wqk[c + h * d:c + (h + 1) * d])], dtype, device, src_channels=cin)
                      for h in range(self.num_heads)]
        if attention_module.position_only or attention_module.position_and_content:
            # per-query position tables of head h: scale * q_h . [rel_height; rel_width] (gma_utils.py:18-30) = a 1x1 layer on
            # `inp` whose weight is [E_h; E_w] @ W_q,h ((2P-1) * 2 rows, folded in fp64), scale applied by the epilogue
            pe = attention_module.pos_emb
            emb = torch.cat([pe.rel_height.weight, pe.rel_width.weight], 0).detach().double()
            self.att_pos = [ops.PackedConv([ConvWeights((emb @ wqk[h * d:(h + 1) * d, :, 0, 0].detach().double()).float()[:, :, None, None])],
                                           dtype, device, src_channels=cin) for h in range(self.num_heads)]
            self.max_pos = pe.rel_height.weight.shape[0] // 2 + 1
        return to_v, proj

    # -- run --------------------------------------------------------------------------------
    def make_cfg(self, B: int, H: int, W: int, iters: int, out_hw, pad, alternate_corr: bool, feat_dim: int, volume_layout: int = 0,
                 fork_flow: bool = False) -> _lib.RaftCfg:
        return _lib.RaftCfg(self.variant, dtype_code(self.dtype), B, H, W, feat_dim, self.corr_levels, self.corr_radius,
                            self.hidden_dim, self.context_dim, iters, int(alternate_corr), out_hw[0], out_hw[1], pad[0], pad[1],
                            self.impl, 0 if alternate_corr else int(volume_layout), int(fork_flow), self.num_heads)

    def volume_tiled(self, fmap1: torch.Tensor, impl: int = 0) -> bool:
        """Whether build_volume gives the tiled pyramid for these features: f16 / bf16 with tensor-core-shaped features and a
        (radius, levels) pair the tiled lookup is instantiated for."""
        return _TILED and impl != 1 and self.corr_radius in (3, 4) and ops.tiled_supported(fmap1, self.corr_levels) \
            and (self.corr_radius, self.corr_levels) in ((4, 4), (4, 3), (4, 2), (4, 1), (3, 4), (3, 3))

    def build_volume(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """(a1 + a2 pyramid, its layout) for the refinement loop of this engine: the tiled pyramid (layout 1: 64-byte tiles,
        csrc/corr_tiled.cu) where volume_tiled says so, else the dense one (layout 0)."""
        if self.volume_tiled(fmap1, impl):
            return ops.corr_volume_build_tiled(fmap1, fmap2, self.corr_levels), 1
        return ops.corr_volume_build(fmap1, fmap2, self.corr_levels, impl=impl), 0

    def before_loop(self, pyramid: Sequence[torch.Tensor], coords: torch.Tensor) -> Sequence[torch.Tensor]:
        """What the loop reads, from what build_volume returned, once the engine has adjusted the start coordinates (fp32 [B,H,W,2], in
        place) after the volume exists.  The pyramid unchanged, and no launch, for every model but CSFlow."""
        return pyramid

    def _new_workspace(self, cfg: _lib.RaftCfg) -> torch.Tensor:
        nbytes = getattr(load(), self._ws_symbol)(C.byref(cfg))
        if nbytes == 0:
            check(-1, self._ws_symbol[4:])
        return torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    def workspace(self, cfg: _lib.RaftCfg, scratch: Optional[dict] = None) -> torch.Tensor:
        if scratch is not None:
            # the caller owns the scratch memory (a CUDA graph keeps the workspace it was captured with alive)
            key = ("raft_ws", cfg.B, cfg.H, cfg.W)
            ws = scratch.get(key)
            if ws is None:
                ws = scratch[key] = self._new_workspace(cfg)
            return ws
        # one workspace per CUDA stream (batches in flight on different streams must not share scratch memory,
        # ptlflow_b200/pipeline.py) and, per stream, one shape resident (bounded memory, SURVEY appendix B.7)
        sid = torch.cuda.current_stream(self.device).cuda_stream
        key = (cfg.B, cfg.H, cfg.W)
        ent = self._workspaces.get(sid)
        if ent is None or ent[0] != key:
            ent = (key, self._new_workspace(cfg))
            if len(self._workspaces) >= 8:
                # streams come and go: do not grow without bound.  A dropped tensor returns to torch's caching allocator,
                # which keeps the block reserved for the stream it was allocated on until that stream's queued work is
                # done -- an evicted workspace with work still in flight is therefore not reused under that work.
                self._workspaces.pop(next(iter(self._workspaces)))
            self._workspaces[sid] = ent
        return ent[1]

    def _call(self, symbol: str, cfg: _lib.RaftCfg, weights, ws: torch.Tensor, pyramid: Optional[Sequence[torch.Tensor]], net: torch.Tensor,
              inp: torch.Tensor, coords: torch.Tensor, *args, fmap1: Optional[torch.Tensor] = None, flow_up: Optional[torch.Tensor] = None,
              flow_small: Optional[torch.Tensor] = None, attention: Optional[torch.Tensor] = None) -> None:
        """``symbol(cfg, weights, buffers, *args, stream)`` on the current stream of the engine's device."""
        pyr = ptr_array(pyramid) if pyramid is not None else None
        buf = _lib.RaftBuffers(C.cast(pyr, C.POINTER(C.c_void_p)) if pyr is not None else None, _ptr(fmap1), net.data_ptr(), inp.data_ptr(),
                               coords.data_ptr(), _ptr(flow_up), _ptr(flow_small), ws.data_ptr(), ws.numel(), _ptr(attention), self.agg_gamma,
                               _ptr(self.agg_score), self.pool_min_side)
        with torch.cuda.device(self.device):
            check(getattr(load(), symbol)(C.byref(cfg), C.byref(weights), C.byref(buf), *args, stream_ptr(self.device)), symbol[4:])

    def _scale_weights(self, scale: int):
        return self.weights  # one update block serves every scale

    def _iter_args(self, corr_scale: float) -> tuple:
        return ()  # the update_iter entry point's arguments after the mask

    def refine(self, pyramid: Sequence[torch.Tensor], layout: int, net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, iters: int,
               out_hw, pad, fmap1: Optional[torch.Tensor] = None, attention: Optional[torch.Tensor] = None, scratch: Optional[dict] = None,
               fork_flow: bool = False):
        """Runs the loop in place on (net, coords) over ``pyramid`` (of ``layout``, as build_volume returned them; the feature pyramid
        of fmap2 when ``fmap1`` is given); returns (flow_up fp32 [B,2,oh,ow], flow_small fp32 [B,2,H,W])."""
        B, H, W, _ = net.shape
        cfg = self.make_cfg(B, H, W, iters, out_hw, pad, fmap1 is not None, fmap1.shape[-1] if fmap1 is not None else 0, layout, fork_flow)
        ws = self.workspace(cfg, scratch)
        flow_up = torch.empty((B, 2, out_hw[0], out_hw[1]), dtype=torch.float32, device=self.device)
        flow_small = torch.empty((B, 2, H, W), dtype=torch.float32, device=self.device)
        self._call(self._refine_symbol, cfg, self.weights, ws, pyramid, net, inp, coords, fmap1=fmap1, flow_up=flow_up, flow_small=flow_small,
                   attention=attention)
        return flow_up, flow_small

    def update_iter(self, net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, corr: Optional[torch.Tensor] = None,
                    pyramid: Optional[Sequence[torch.Tensor]] = None, want_mask: bool = False, attention: Optional[torch.Tensor] = None,
                    fmap1: Optional[torch.Tensor] = None, corr_scale: float = 0.0, scale: int = 0):
        """One update-block evaluation of scale ``scale`` (operator-level tests).  corr: pixel-major [B,H,W,planes]; attention (gma):
        head-major [heads*B*N, N]; returns the [B,H,W,9*upsample**2] mask when asked (raft_small has no mask head)."""
        B, H, W, _ = net.shape
        up = self.upsample
        cfg = self.make_cfg(B, H, W, 1, (up * H, up * W), (0, 0), fmap1 is not None, fmap1.shape[-1] if fmap1 is not None else 0)
        ws = self.workspace(cfg)
        has_mask = want_mask and self.variant != _lib.VARIANT_RAFT_SMALL  # SmallUpdateBlock has no mask head
        mask = torch.empty((B, H, W, 9 * up * up), dtype=self.dtype, device=self.device) if has_mask else None
        self._call(self._iter_symbol, cfg, self._scale_weights(scale), ws, pyramid, net, inp, coords, _ptr(corr), _ptr(mask),
                   *self._iter_args(corr_scale), fmap1=fmap1, attention=attention)
        return mask


def _align(n: int, a: int) -> int:
    return (n + a - 1) // a * a


def _pad_conv(conv: torch.nn.Module, cout: int, cin: int) -> ConvWeights:
    """conv's weight / bias zero-padded to [cout, cin, kh, kw] / [cout]."""
    w = conv.weight.detach()
    wp = torch.zeros((cout, cin) + tuple(w.shape[2:]), dtype=w.dtype, device=w.device)
    wp[: w.shape[0], : w.shape[1]] = w
    b = None
    if conv.bias is not None:
        b = torch.zeros(cout, dtype=conv.bias.dtype, device=conv.bias.device)
        b[: conv.bias.shape[0]] = conv.bias.detach()
    return ConvWeights(wp, b)


class SKFlowEngine(RaftEngine):
    """SKFlow's update block (skflow/update.py:7-99) packed for pfb_skflow_refine: every PCBlock's 1x1 layers through
    ops.PackedConv, its depthwise filters as fp32 [k*k][C], all channel counts zero-padded to multiples of 32 (the padding stays
    exactly zero through the block).  The attention is GMA's."""

    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_skflow_workspace_bytes", "pfb_skflow_refine", "pfb_skflow_update_iter"

    def _pack(self, update_block: torch.nn.Module, attention_module: Optional[torch.nn.Module] = None) -> _lib.SkflowWeights:
        ub = update_block
        enc = ub.encoder
        planes = self.corr_levels * (2 * self.corr_radius + 1) ** 2
        w = _lib.SkflowWeights()
        blocks = ((_lib.SK_CONVC1, enc.convc1, planes), (_lib.SK_CONVC2, enc.convc2, 256), (_lib.SK_CONVF2, enc.convf2, 128),
                  (_lib.SK_CONV, enc.conv, 256), (_lib.SK_GRU, ub.gru, 512), (_lib.SK_FLOW_HEAD, ub.flow_head, 128))
        for bid, blk, cin in blocks:
            w.blocks[bid] = self._pack_block(blk, cin)
        self.corr_stride = _align(planes, 32)  # the lookup buffer: planes channels, zero up to the padded width
        for name, conv, srcs in (("convf1", enc.convf1, None), ("mask1", ub.mask[0], [128]), ("mask2", ub.mask[2], [256])):
            setattr(w, name, self._conv(conv, srcs))
        to_v, proj = self._pack_attention(ub.aggregator, attention_module)
        w.agg_v = self._layer(to_v)
        if proj is not None:
            w.agg_proj = self._layer(proj)
        return w

    def _pack_block(self, blk: torch.nn.Module, cin: int) -> _lib.PcBlock:
        """PCBlock4_Deep_nopool_res(cin, cout, k_conv) -> pfb_pc_block (C = align(cin, 32), hid = align(int(1.5 cin), 32))."""
        device = self.device
        C, hid = _align(cin, 32), _align(int(1.5 * cin), 32)
        cout = blk.ffn2[2].weight.shape[0]
        k = _lib.PcBlock()
        k.ffn1a = self._conv(_pad_conv(blk.ffn1[0], hid, C), [C])
        k.ffn1b = self._conv(_pad_conv(blk.ffn1[2], C, hid), [hid])
        k.pw = self._conv(_pad_conv(blk.pw, C, C), [C])
        k.ffn2a = self._conv(_pad_conv(blk.ffn2[0], hid, C), [C])
        k.ffn2b = self._conv(_pad_conv(blk.ffn2[2], cout, hid), [hid])
        k.C, k.hid = C, hid
        convs = list(blk.conv_list)
        if len(convs) > _lib.PFB_SK_MAX_DW:
            raise ValueError(f"skflow: at most {_lib.PFB_SK_MAX_DW} depthwise convolutions per block, got {len(convs)}")
        k.n_dw = len(convs)
        for i, conv in enumerate(convs):
            ks = conv.weight.shape[-1]
            wt = torch.zeros((ks * ks, C), dtype=torch.float32, device=device)  # [tap][channel]
            wt[:, :cin] = conv.weight.detach().to(device, torch.float32).reshape(cin, ks * ks).t()
            bt = torch.zeros(C, dtype=torch.float32, device=device)
            if conv.bias is not None:
                bt[:cin] = conv.bias.detach().to(device, torch.float32)
            self._keep += [wt, bt]
            k.dw_k[i], k.dw_weight[i], k.dw_bias[i] = ks, wt.data_ptr(), bt.data_ptr()
        return k


class SEARaftEngine(RaftEngine):
    """SEA-RAFT's heads and update block (sea_raft.py:104-133, update.py:18-54, layer.py:41-83) packed for pfb_searaft_refine; built
    from the model (init_conv, flow_head, upsample_weight and, iters > 0, update_block).  Each ConvNextBlock becomes its depthwise
    filter (fp32 [k*k][384]) and two 1x1 layers, folded in fp64 from the parameters: pw1 = pwconv1 with the LayerNorm affine
    (W1 diag(ln_w), b1 + W1 ln_b), and out = final(x + gamma * pwconv2(h)) over the two sources [h | x] ([Wf diag(gamma) W2 | Wf],
    Wf (gamma b2) + bf)."""

    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_searaft_workspace_bytes", "pfb_searaft_refine", "pfb_searaft_update_iter"

    def _pack(self, model: torch.nn.Module) -> _lib.SearaftWeights:
        P = self._conv
        w = _lib.SearaftWeights()
        w.init_conv = P(model.init_conv, [256])
        fh = model.flow_head
        w.flow1 = P(fh[0], [128])
        w2, b2 = fh[2].weight.detach()[:2], fh[2].bias.detach()[:2]  # the flow outputs; info (2:6) feeds training only
        w.flow2 = P(ConvWeights(w2.contiguous(), b2.contiguous()), [256])
        if self.dtype != torch.float32:
            w.flow2t = P(_taps(w2), [256])
        w.mask1 = P(model.upsample_weight[0], [128])
        w.mask2 = P(model.upsample_weight[2], [256])
        w.ln_eps = 1e-6
        ub = getattr(model, "update_block", None)
        if ub is not None:
            enc = ub.encoder
            planes = self.corr_levels * (2 * self.corr_radius + 1) ** 2
            w.convc1, w.convc2 = P(enc.convc1, [planes]), P(enc.convc2, [256])
            w.convf1 = self._layer(_pack_convf1(enc.convf1, self.dtype, self.device))
            w.convf2, w.conv = P(enc.convf2, [128]), P(enc.conv, [256])
            if len(ub.refine) > _lib.PFB_SR_MAX_BLOCKS:
                raise ValueError(f"sea_raft: at most {_lib.PFB_SR_MAX_BLOCKS} ConvNeXt blocks, got {len(ub.refine)}")
            w.num_blocks = len(ub.refine)
            for i, blk in enumerate(ub.refine):
                w.blocks[i] = self._pack_block(blk)
                w.ln_eps = blk.norm.eps
        return w

    def _pack_block(self, blk: torch.nn.Module) -> _lib.ConvNextBlock:
        device = self.device
        f64 = lambda t: t.detach().to(device, torch.float64)  # noqa: E731
        W1, b1, lw, lb = f64(blk.pwconv1.weight), f64(blk.pwconv1.bias), f64(blk.norm.weight), f64(blk.norm.bias)
        W2, b2, g = f64(blk.pwconv2.weight), f64(blk.pwconv2.bias), f64(blk.gamma)
        Wf, bf = f64(blk.final.weight)[:, :, 0, 0], f64(blk.final.bias)
        pw1 = ConvWeights((W1 * lw[None, :]).float()[:, :, None, None].contiguous(), (b1 + W1 @ lb).float())
        out = ConvWeights(torch.cat([Wf @ (g[:, None] * W2), Wf], 1).float()[:, :, None, None].contiguous(), (Wf @ (g * b2) + bf).float())
        C, k = blk.dwconv.weight.shape[0], blk.dwconv.weight.shape[-1]
        dw_w = blk.dwconv.weight.detach().to(device, torch.float32).reshape(C, k * k).t().contiguous()  # [tap][channel]
        dw_b = blk.dwconv.bias.detach().to(device, torch.float32).contiguous()
        self._keep += [dw_w, dw_b]
        b = _lib.ConvNextBlock()
        b.dw_k, b.dw_weight, b.dw_bias = k, dw_w.data_ptr(), dw_b.data_ptr()
        b.pw1 = self._conv(pw1, [C])
        b.out = self._conv(out, [4 * Wf.shape[0], C])
        return b


class MSRaftEngine(RaftEngine):
    """MS-RAFT+'s update block (ms_raft_plus/update.py:119-153: RAFT's BasicUpdateBlock with convc1 over levels * (2r+1)^2 planes and
    a 36-channel mask head) packed exactly as RaftEngine packs raft's, driven one scale at a time through pfb_msraft_refine
    (pfb_raft_cfg variant VARIANT_MS_RAFT_P, 5)."""

    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_msraft_workspace_bytes", "pfb_msraft_refine", "pfb_msraft_update_iter"
    upsample = 2

    def _iter_args(self, corr_scale: float) -> tuple:
        return (corr_scale,)

    def _refine_args(self, corr_scale: float, upflow2: int) -> tuple:
        return (corr_scale,)  # (the loop ends at 1/2 scale: nothing to add to the last convex upsample)

    def refine_scale(self, scale: int, pyramid: Sequence[torch.Tensor], layout: int, net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor,
                     iters: int, out_hw, pad, ws: torch.Tensor, fmap1: Optional[torch.Tensor] = None, corr_scale: float = 0.0, last: bool = False,
                     upflow2: int = 0, fork_flow: bool = False):
        """Scale ``scale`` in place on (net, coords) over ``pyramid`` of ``layout`` (as for refine).  Not last: returns the next scale's
        coordinates fp32 [B,2H,2W,2].  Last: returns (flow_up fp32 [B,2,oh,ow], flow_small fp32 [B,2,oh//16,ow//16]), with ``upflow2``
        bilinear 2x steps after the convex upsample."""
        B, H, W, _ = net.shape
        cfg = self.make_cfg(B, H, W, iters, out_hw, pad, fmap1 is not None, fmap1.shape[-1] if fmap1 is not None else 0, layout, fork_flow)
        flow_up = flow_small = nxt = None
        if last:
            flow_up = torch.empty((B, 2, out_hw[0], out_hw[1]), dtype=torch.float32, device=self.device)
            flow_small = torch.empty((B, 2, out_hw[0] // 16, out_hw[1] // 16), dtype=torch.float32, device=self.device)
        else:
            nxt = torch.empty((B, 2 * H, 2 * W, 2), dtype=torch.float32, device=self.device)
        self._call(self._refine_symbol, cfg, self._scale_weights(scale), ws, pyramid, net, inp, coords, *self._refine_args(corr_scale, upflow2),
                   _ptr(nxt), fmap1=fmap1, flow_up=flow_up, flow_small=flow_small)
        return (flow_up, flow_small) if last else nxt


class CCMREngine(MSRaftEngine):
    """CCMR's update block (ccmr/update.py:110-168: MS-RAFT+'s layers with a GMA-width GRU over [inp | motion | motion_global]) packed
    as RaftEngine packs gma's, plus per scale the XCiT of the context (``xcit[i]``) and the aggregator (``update_block.aggregator[i]``)
    as pfb_xcit_block descriptors, folded in fp64 (xcit.py:242-300): norm1's affine into q | k and v, gamma1 into proj, gamma3 into
    LPI's second convolution, norm2's affine into fc1 and gamma2 into fc2.  Driven one scale at a time through pfb_ccmr_refine
    (pfb_raft_cfg variant VARIANT_CCMR, 6)."""

    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_ccmr_workspace_bytes", "pfb_ccmr_refine", "pfb_ccmr_update_iter"

    def _pack(self, update_block: torch.nn.Module, xcit: Optional[torch.nn.Module] = None) -> _lib.RaftWeights:
        raft = super()._pack(update_block)
        self.scale_weights = []
        for i in range(len(update_block.aggregator)):
            w = _lib.CcmrWeights()
            w.raft = raft
            w.context = self._pack_xcit(xcit[i], separate=False)
            w.aggregator = self._pack_xcit(update_block.aggregator[i], separate=True)
            self.scale_weights.append(w)
        return raft

    def _scale_weights(self, scale: int):
        return self.scale_weights[scale]

    def _refine_args(self, corr_scale: float, upflow2: int) -> tuple:
        return (corr_scale, int(upflow2))

    def _pack_xcit(self, xc: torch.nn.Module, separate: bool) -> _lib.XcitBlock:
        device = self.device
        blk = xc.blocks[0]
        f64 = lambda t: t.detach().to(device, torch.float64)  # noqa: E731
        f32 = lambda t: self._hold(t.float().contiguous())  # noqa: E731
        C = blk.norm1.weight.shape[0]
        ln1w, ln1b = f64(blk.norm1.weight), f64(blk.norm1.bias)
        a = blk.attn
        if separate:
            wqk, wv = f64(a.to_qk.weight), f64(a.to_v.weight)
            bqk = f64(a.to_qk.bias) if a.to_qk.bias is not None else torch.zeros(2 * C, dtype=torch.float64, device=device)
            bv = f64(a.to_v.bias) if a.to_v.bias is not None else torch.zeros(C, dtype=torch.float64, device=device)
        else:
            wqkv = f64(a.qkv.weight)
            bqkv = f64(a.qkv.bias) if a.qkv.bias is not None else torch.zeros(3 * C, dtype=torch.float64, device=device)
            wqk, wv, bqk, bv = wqkv[: 2 * C], wqkv[2 * C:], bqkv[: 2 * C], bqkv[2 * C:]
        g1, g2, g3 = f64(blk.gamma1), f64(blk.gamma2), f64(blk.gamma3)

        def P(weight, bias, cin):  # a folded linear as a 1x1 layer
            return self._conv(ConvWeights(weight.float()[:, :, None, None].contiguous(), bias.float().contiguous()), [cin])

        def dw(conv, scale):  # [C,1,3,3] -> fp32 [9][C] tap-major, times a per-channel scale
            w = f64(conv.weight).reshape(C, 9) * scale[:, None]
            return f32(w.t()), f32(f64(conv.bias) * scale)

        x = _lib.XcitBlock()
        tp = xc.pos_embeder.token_projection
        x.pos_proj = P(f64(tp.weight)[:, :, 0, 0], f64(tp.bias), tp.weight.shape[1])
        x.qk = P(wqk * ln1w[None, :], bqk + wqk @ ln1b, C)
        x.v_weight, x.v_bias = f32(wv * ln1w[None, :]), f32(bv + wv @ ln1b)
        wp, bp = f64(a.proj.weight), f64(a.proj.bias)
        x.proj_weight, x.proj_bias = f32(g1[:, None] * wp), f32(g1 * bp)
        x.temperature = f32(f64(a.temperature).reshape(-1))
        x.ln3_weight, x.ln3_bias = f32(f64(blk.norm3.weight)), f32(f64(blk.norm3.bias))
        lp = blk.local_mp
        one = torch.ones(C, dtype=torch.float64, device=device)
        x.dw1_weight, x.dw1_bias = dw(lp.conv1, one)
        x.gn_weight, x.gn_bias = f32(f64(lp.bn.weight)), f32(f64(lp.bn.bias))
        x.dw2_weight, x.dw2_bias = dw(lp.conv2, g3)
        w1, b1, ln2w, ln2b = f64(blk.mlp.fc1.weight), f64(blk.mlp.fc1.bias), f64(blk.norm2.weight), f64(blk.norm2.bias)
        x.fc1 = P(w1 * ln2w[None, :], b1 + w1 @ ln2b, C)
        x.fc2 = P(g2[:, None] * f64(blk.mlp.fc2.weight), g2 * f64(blk.mlp.fc2.bias), w1.shape[0])
        x.ln_eps, x.gn_eps = float(blk.norm1.eps), float(lp.bn.eps)
        return x

    def _hold(self, t: torch.Tensor) -> int:
        self._keep.append(t)
        return t.data_ptr()

    def xcit_context(self, scale: int, inp: torch.Tensor) -> torch.Tensor:
        """global_context = xcit[scale](inp) (operator-level tests): inp, result pixel-major [B,H,W,128]."""
        B, H, W, _ = inp.shape
        cfg = self.make_cfg(B, H, W, 1, (2 * H, 2 * W), (0, 0), False, 0)
        ws = self.workspace(cfg)
        out = torch.empty_like(inp)
        with torch.cuda.device(self.device):
            check(load().pfb_xcit_context(C.byref(cfg), C.byref(self.scale_weights[scale]), inp.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                          ws.numel(), stream_ptr(self.device)), "xcit_context")
        return out


def sine_position(H: int, W: int, C: int, device) -> torch.Tensor:
    """PositionEmbeddingSine(C // 2) of an H x W grid (flow1d/position.py), fp32 pixel-major [H, W, C]: channels 0 .. C/2-1 from the
    row, C/2 .. C-1 from the column; inside each half sin at even and cos at odd channels of (i + 1) / (n + 1e-6) * 2 pi / dim_t,
    dim_t[j] = 10000 ** (2 (j // 2) / (C / 2))."""
    npf = C // 2
    dim_t = 10000.0 ** (2 * (torch.arange(npf, dtype=torch.float32, device=device) // 2) / npf)

    def half(n: int) -> torch.Tensor:  # [n, npf]
        e = torch.arange(1, n + 1, dtype=torch.float32, device=device) / (n + 1e-6) * (2 * math.pi)
        p = e[:, None] / dim_t
        return torch.stack((p[:, 0::2].sin(), p[:, 1::2].cos()), dim=2).flatten(1)

    return torch.cat((half(H)[:, None, :].expand(H, W, npf), half(W)[None, :, :].expand(H, W, npf)), dim=2).contiguous()


class Flow1DEngine(RaftEngine):
    """Flow1D (flow1d.py:148-246): RAFT's update block over the 2 (2r+1) planes of the 1D lookup, run by pfb_raft_refine as
    pfb_raft_cfg variant VARIANT_FLOW1D (7), and, in place of the correlation pyramid, the four 1D attentions and the two 1D volumes
    (build_volume).
    The attentions' query / key 1x1 convolutions are packed here; ``x + pos`` is one add in the storage type ahead of each (the
    reference's rounding of its half model)."""

    def _pack(self, update_block: torch.nn.Module, attention: Sequence[torch.nn.Module] = ()) -> _lib.RaftWeights:
        w = super()._pack(update_block)
        self.proj: Dict[str, ops.PackedConv] = {}
        for axis, mod in zip("xy", attention):
            for sub, m in (("self_", mod.self_attn), ("", mod)):
                for kind in ("query", "key"):
                    conv = getattr(m, kind + "_conv")
                    self.proj[f"{axis}.{sub}{kind}"] = ops.PackedConv([conv], self.dtype, self.device, src_channels=[conv.in_channels])
        self._pos: Dict[Tuple[int, int, int], torch.Tensor] = {}
        return w

    def position(self, H: int, W: int, C: int) -> torch.Tensor:
        """sine_position in the storage type (computed in fp32 and rounded once), cached per grid."""
        key = (H, W, C)
        pos = self._pos.get(key)
        if pos is None:
            if len(self._pos) >= 8:
                self._pos.pop(next(iter(self._pos)))
            pos = self._pos[key] = sine_position(H, W, C, self.device).to(self.dtype)
        return pos

    def attention_features(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """(feature2_x, feature2_y) of flow1d.py:176, 184: attn_x = column self-attention of fmap1, then its row attention into fmap2;
        attn_y = row self-attention, then column attention (attention.py:40-78).  Pixel-major [B,H,W,C] in, out."""
        B, H, W, C = fmap1.shape
        pos = self.position(H, W, C)
        f1p, f2p = fmap1 + pos, fmap2 + pos

        def proj(name: str, x: torch.Tensor) -> torch.Tensor:
            return ops.conv2d([x], self.proj[name], torch.empty_like(x), impl=impl)

        def attend(prefix: str, q_in: torch.Tensor, k_in: torch.Tensor, v: torch.Tensor, axis: int) -> torch.Tensor:
            return ops.attn1d(proj(prefix + "query", q_in), proj(prefix + "key", k_in), v, axis, impl=impl)

        f2_x = attend("x.", attend("x.self_", f1p, f1p, fmap1, 1) + pos, f2p, fmap2, 0)
        f2_y = attend("y.", attend("y.self_", f1p, f1p, fmap1, 0) + pos, f2p, fmap2, 1)
        return f2_x, f2_y

    def build_volume(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """([corr_x [B*H*W, W], corr_y [B*H*W, H]], layout 0): corr_x of fmap1 against feature2_y along rows, corr_y against
        feature2_x along columns, both scaled by 1/sqrt(C) (flow1d.py:177-190, correlation.py:77-107)."""
        f2_x, f2_y = self.attention_features(fmap1, fmap2, impl)
        return [ops.attn1d(fmap1, f2_y, None, 0, _lib.ATTN1D_CORR, impl=impl), ops.attn1d(fmap1, f2_x, None, 1, _lib.ATTN1D_CORR, impl=impl)], 0


def fold_conv_bn_relu(block: torch.nn.Module) -> ConvWeights:
    """A ConvBNReLU (csflow.py:299-319: a convolution without bias, then eval-mode BatchNorm) as one convolution with bias, folded in
    fp64: w' = w s, b' = beta - mean s, s = gamma / sqrt(var + eps).  The ReLU is the convolution's epilogue."""
    conv, bn = block.conv, block.bn
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    w = conv.weight.detach().double() * s[:, None, None, None]
    b = bn.bias.detach().double() - bn.running_mean.detach().double() * s
    return ConvWeights(w.float().contiguous(), b.float())


def csflow_convc1_permutation(levels: int, radius: int) -> torch.Tensor:
    """Column b of the lookup buffer ([4D taps of levels 0..L-1 | strip taps of levels 0..L-1]) is input column perm[b] of the
    reference's convc1, whose input interleaves the two channels per level ([4D l | strip l], csflow.py:488-492)."""
    kk = (2 * radius + 1) ** 2
    t = torch.arange(kk)
    return torch.cat([l * 2 * kk + ch * kk + t for ch in (0, 1) for l in range(levels)])


class CSFlowEngine(RaftEngine):
    """CSFlow (csflow.py:116-278, 445-493): RAFT's update block over [4D taps | strip taps], run by pfb_raft_refine as pfb_raft_cfg
    variant VARIANT_CSFLOW (8).  Packs the four ConvBNReLU blocks of the strip module (BatchNorm folded) and convc1 with its input
    columns permuted to the lookup buffer's order; build_volume adds the strip maps to RAFT's pyramid, and before_loop turns them into
    the separable fp32 tables the loop reads while adding the initial strip flow to the coordinates."""

    def _pack(self, update_block: torch.nn.Module, strip_block: Optional[torch.nn.Module] = None) -> _lib.RaftWeights:
        w = super()._pack(update_block)
        c1 = update_block.encoder.convc1
        perm = csflow_convc1_permutation(self.corr_levels, self.corr_radius).to(c1.weight.device)
        pc = ops.PackedConv([ConvWeights(c1.weight.detach()[:, perm].contiguous(), c1.bias)], self.dtype, self.device,
                            src_channels=[c1.in_channels])
        self.layers[_lib.L_CONVC1] = pc
        w.layers[_lib.L_CONVC1] = pc.layer_struct()
        self.strip = {name: ops.PackedConv([fold_conv_bn_relu(getattr(strip_block, name))], self.dtype, self.device, src_channels=[256])
                      for name in ("conv1_1", "conv1_2", "conv2_1", "conv2_2")}
        return w

    def strip_maps(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """(sw [B*H*W, 1, W], sh [B*H*W, H, 1]) of StripCrossCorrMap_v2 (csflow.py:239-278), in the storage type, unscaled."""
        def cbr(name: str, x: torch.Tensor) -> torch.Tensor:
            return ops.conv2d([x], self.strip[name], torch.empty_like(x), _lib.EPI_RELU, impl=impl)

        kw, kh = ops.strip_means(cbr("conv2_1", fmap2), cbr("conv2_2", fmap2))
        sw = ops.corr_volume_build_ex(cbr("conv1_1", fmap1), kw, 1, scale=1.0, impl=impl)[0]
        sh = ops.corr_volume_build_ex(cbr("conv1_2", fmap1), kh, 1, scale=1.0, impl=impl)[0]
        return sw, sh

    def build_volume(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """(RaftEngine's pyramid (dense or tiled) + [sw, sh], its layout)."""
        pyr, layout = super().build_volume(fmap1, fmap2, impl)
        return list(pyr) + list(self.strip_maps(fmap1, fmap2, impl)), layout

    def before_loop(self, pyramid: Sequence[torch.Tensor], coords: torch.Tensor) -> List[torch.Tensor]:
        L = self.corr_levels
        _, H, W, _ = coords.shape
        tab_w, tab_h = ops.strip_prepare(pyramid[L], pyramid[L + 1], (H, W), L, coords)
        return list(pyramid[:L]) + [tab_w, tab_h]


class SCVEngine(RaftEngine):
    """SCV (scv.py:148-500): RAFT's BasicUpdateBlock over the 405-plane sparse lookup, run by pfb_raft_refine as pfb_raft_cfg variant
    VARIANT_SCV8 (9) or VARIANT_SCV4 (10, convex 4x).  build_volume keeps the num_k best matches of every query (pfb_knn_topk, the
    volume never materialised); before_loop turns them into the fp32 table the loop's lookup reads, with the warm start folded in."""

    def _pack(self, update_block: torch.nn.Module, num_k: int = 32) -> _lib.RaftWeights:
        self.num_k = num_k
        self.upsample = 4 if self.variant == _lib.VARIANT_SCV4 else 8
        return super()._pack(update_block)

    def make_cfg(self, B: int, H: int, W: int, iters: int, out_hw, pad, alternate_corr: bool, feat_dim: int, volume_layout: int = 0,
                 fork_flow: bool = False) -> _lib.RaftCfg:
        # feat_dim carries num_k for the sparse lookup (include/ptlflow_b200.h, a21)
        return super().make_cfg(B, H, W, iters, out_hw, pad, False, self.num_k, 0, fork_flow)

    def build_volume(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """([val fp32 [B*N, k], idx int32 [B*N, k]], layout 0): the k-NN of compute_sparse_corr (scv.py:48-83), scaled by 1/sqrt(C)."""
        # fp32 features have no tensor-core path: every impl runs the exact SIMT kernel, as for the convolutions
        impl = 1 if fmap1.dtype == torch.float32 else impl
        return list(ops.knn_topk(fmap1, fmap2, self.num_k, 1.0 / math.sqrt(fmap1.shape[-1]), impl=impl)), 0

    def before_loop(self, pyramid: Sequence[torch.Tensor], coords: torch.Tensor) -> List[torch.Tensor]:
        return [ops.sparse_prepare(pyramid[0], pyramid[1], coords)]


class LLAFlowEngine(RaftEngine):
    """LLA-Flow (llaflow.py:140-217): GMA's loop (PFB_VARIANT_GMA, llaflow) or RAFT's (PFB_VARIANT_RAFT, llaflow_raft) over a volume with
    the local-attention terms of aggregate.py.  Packs the stacked ls1 | ls2 query / key convolution (N = 512), lsa.to_v and s_lsa.to_f1 /
    to_f2, and reads both gammas once; lla_volume builds the volume from (fmap1, fmap2, inp) as one K = 6656 GEMM (csrc/llaflow.cu)."""

    def _pack(self, update_block: torch.nn.Module, attention_module: Optional[torch.nn.Module] = None, local=None) -> _lib.RaftWeights:
        w = super()._pack(update_block, attention_module)
        ls1, ls2, lsa, s_lsa, gamma = local

        def P(convs, cin: int) -> ops.PackedConv:
            return ops.PackedConv(convs, self.dtype, self.device, src_channels=[cin])

        self.ls_qk = P([ls1.to_qk, ls2.to_qk], ls1.to_qk.in_channels)
        self.lsa_v, self.to_f1, self.to_f2 = P([lsa.to_v], 256), P([s_lsa.to_f1], 256), P([s_lsa.to_f2], 256)
        self.lsa_gamma = float(lsa.gamma.detach().float().cpu().item())
        self.gamma = float(gamma.detach().float().cpu().item())
        return w

    def lla_volume(self, fmap1: torch.Tensor, fmap2: torch.Tensor, inp: torch.Tensor, impl: int = 0):
        """(pyramid, layout) of corr.py:13-27 with corr2 of ShiftLSA: the tiled pyramid from pfb_shift_volume_tiled where RaftEngine's
        volume_tiled holds for fmap1, else the dense pyramid of A' and the materialised B' on pfb_corr_volume_build_ex (SIMT: the
        tensor-core volume takes C <= 256)."""
        B, H, W, C = fmap1.shape

        def conv(packed: ops.PackedConv, x: torch.Tensor) -> torch.Tensor:
            return ops.conv2d([x], packed, torch.empty((B, H, W, packed.Cout), dtype=x.dtype, device=x.device), impl=impl)

        a1, a2 = ops.local_similar(conv(self.ls_qk, inp))
        fmap2p = ops.local_aggregate(fmap2, conv(self.lsa_v, fmap2), a2, self.lsa_gamma)
        tiled = self.volume_tiled(fmap1, impl)
        a, b = ops.shift_pack(fmap1, conv(self.to_f1, fmap1), a1, fmap2p, conv(self.to_f2, fmap2p), self.gamma, padded=tiled)
        if tiled:
            return ops.shift_volume_tiled(a, b, self.corr_levels), 1
        return ops.corr_volume_build_ex(a, b, self.corr_levels, scale=1.0, impl=1), 0


class CRAFTEngine(RaftEngine):
    """CRAFT (craft.py:57-376): GMA's loop (PFB_VARIANT_GMA) with the intra-frame modes as its heads, and the three cross-attention
    sites of setrans.py.  The aggregator (ExpandedFeatTrans: first_linear, feat_softaggr, input_skip_coeff) rides on GMA's multi-head
    aggregate: first_linear is to_v, each mode's attn @ v lands in its 128 columns, and pfb_craft_mode_aggregate (agg_score =
    feat2score, agg_gamma = input_skip_coeff) replaces project + AXPY.  Each attention's q / k projections are packed per mode as 1x1
    layers with head-major outputs (the intra-frame 32-channel modes zero-padded to 64, which leaves every dot product unchanged)."""

    def _pack(self, update_block: torch.nn.Module, attention_module=None, f2_trans=None, corr_trans=None) -> _lib.RaftWeights:
        w = super()._pack(update_block, attention_module)
        self.f2 = self._pack_setrans(f2_trans)
        self.corr = self._pack_setrans(corr_trans) if corr_trans is not None else None
        if corr_trans is not None:  # the shared q = k projection of all modes at once (the fused volume's operands)
            lin = corr_trans.setrans.query
            self.corr_qk = ops.PackedConv([ConvWeights(lin.weight.detach()[:, :, None, None], lin.bias)], self.dtype, self.device,
                                          src_channels=[lin.weight.shape[1]])
        ft = f2_trans.setrans.out_trans
        self.f2_v = ops.PackedConv([ConvWeights(ft.first_linear.weight.detach()[:, :, None, None])], self.dtype, self.device, src_channels=[256])
        self.f2_score = ft.feat_softaggr.feat2score.weight.detach().to(self.device, torch.float32).reshape(-1).contiguous()
        self.f2_coeff = float(ft.input_skip_coeff.detach().float().cpu().item())
        return w

    def _pack_attention(self, agg: torch.nn.Module, attention_module: torch.nn.Module):
        self.num_heads = agg.num_modes
        to_v = ops.PackedConv([ConvWeights(agg.first_linear.weight.detach()[:, :, None, None])], self.dtype, self.device, src_channels=[128])
        self.agg_gamma = float(agg.input_skip_coeff.detach().float().cpu().item())
        self.agg_score = agg.feat_softaggr.feat2score.weight.detach().to(self.device, torch.float32).reshape(-1).contiguous()
        self.att = self._pack_setrans(attention_module)
        return to_v, None

    def _pack_setrans(self, mod: torch.nn.Module) -> dict:
        """A SelfAttVisPosTrans / TransCorrBlock: per mode the q and k 1x1 layers (K = mode width padded to a multiple of 64, zero rows),
        the weighted window bias fp32 [(2R+1)^2], the mode count and width, the position weight and the scalar of attn_softaggr."""
        st = mod.setrans
        M, cin = st.num_modes, st.query.weight.shape[1]
        d = cin // M
        dp = _align(d, 64)

        def per_mode(lin: torch.nn.Linear):
            out = []
            for m in range(M):
                wm = torch.zeros((dp, cin), dtype=lin.weight.dtype, device=lin.weight.device)
                wm[:d] = lin.weight.detach()[m * d:(m + 1) * d]
                b = None
                if lin.bias is not None:
                    b = torch.zeros(dp, dtype=lin.bias.dtype, device=lin.bias.device)
                    b[:d] = lin.bias.detach()[m * d:(m + 1) * d]
                out.append(ops.PackedConv([ConvWeights(wm[:, :, None, None].contiguous(), b)], self.dtype, self.device, src_channels=[cin]))
            return out

        bias = (st.pos_code_weight * mod.vispos_encoder.pos_coder.biases.detach().double()).float().to(self.device).reshape(-1).contiguous()
        soft = getattr(st, "attn_softaggr", None)
        return dict(q=per_mode(st.query), k=per_mode(st.key), M=M, d=d, dp=dp, R=mod.vispos_encoder.pos_coder.R, bias=bias,
                    a=float(soft.feat2score.weight.detach().float().cpu().item()) if soft is not None else 0.0)

    def _scores(self, sp: dict, x1: torch.Tensor, x2: torch.Tensor, impl: int) -> torch.Tensor:
        """Head-major per-mode scores [M*B*N, N] = <q_m(x1), k_m(x2)> / sqrt(d)."""
        B, H, W, _ = x1.shape
        M, dp = sp["M"], sp["dp"]
        q = torch.empty((M, B, H, W, dp), dtype=x1.dtype, device=x1.device)
        k = torch.empty_like(q)
        for m in range(M):
            ops.conv2d([x1], sp["q"][m], q[m], impl=impl)
            ops.conv2d([x2], sp["k"][m], k[m], impl=impl)
        return ops.corr_volume_build_ex(q.view(M * B, H, W, dp), k.view(M * B, H, W, dp), 1, scale=sp["d"] ** -0.5, impl=impl)[0].view(
            M * B * H * W, H * W)

    def attention_probs(self, sp: dict, xn: torch.Tensor, mask_radius: int, impl: int) -> torch.Tensor:
        """CrossAttFeatTrans's softmax probabilities of the normalised tokens xn with themselves (setrans.py:578-648), head-major
        [M*B*N, N]."""
        _, H, W, _ = xn.shape
        logits = self._scores(sp, xn, xn, impl)
        return ops.craft_window_softmax(logits, H, W, sp["bias"], sp["R"], ops.craft_clamp_flag(logits), mask_radius)

    def attend_values(self, attn: torch.Tensor, v: torch.Tensor, F_: int, impl: int = 0) -> torch.Tensor:
        """out[b, i, m F + c] = sum_j attn[m, b, i, j] v[b, j, m F + c]: per mode a 1x1 GEMM over the N attention columns whose weights
        are the sample's v, as the loop's GMA aggregate runs it (one launch for all samples on wgmma, via v's transpose)."""
        B, H, W, MF = v.shape
        M, N = MF // F_, H * W
        out = torch.empty_like(v)
        a = attn.view(M, B, H, W, N)
        tensor = v.dtype != torch.float32 and impl != 1 and N % 8 == 0
        vT = ops.transpose_pm(v.view(B, N, MF), _align(N, 64)) if tensor else None
        zero_bias = torch.zeros(128, dtype=torch.float32, device=v.device)
        for c0 in range(0, MF, 128):  # 128 output columns per GEMM, as for GMA's heads; weight rows strided by M F
            src = a[c0 // F_]
            if tensor:
                layer = ops.PerSampleWeights(v[0].view(N, MF)[:, c0:], zero_bias, 128, MF, v.dtype, vT[0, c0:], vT.shape[-1], 128)
                ops.conv2d([src], layer, out, out_offset=c0, impl=2, w_rows_per_sample=MF)
            else:
                for b in range(B):
                    layer = ops.PerSampleWeights(v[b].view(N, MF)[:, c0:], zero_bias, 128, MF, v.dtype)
                    ops.conv2d([src[b:b + 1]], layer, out[b:b + 1], out_offset=c0, impl=impl)
        return out

    def f2_transform(self, fmap2: torch.Tensor, mask_radius: int = -1, impl: int = 0) -> torch.Tensor:
        """SelfAttVisPosTrans "F2 transformer" (setrans.py:656-710, 346-471): LN(coeff x + soft-aggregate_m(P_m @ V_m)), x = LN(fmap2)."""
        x = ops.layernorm(fmap2, eps=1e-12)
        attn = self.attention_probs(self.f2, x, mask_radius, impl)
        v = ops.conv2d([x], self.f2_v, torch.empty(x.shape[:3] + (self.f2_v.Cout,), dtype=x.dtype, device=x.device), impl=impl)
        y = self.attend_values(attn, v, 256, impl)
        return ops.craft_mode_aggregate(y, self.f2["M"], self.f2_score, self.f2_coeff, x)

    def craft_volume(self, fmap1: torch.Tensor, fmap2t: torch.Tensor, impl: int = 0):
        """(pyramid, layout) of TransCorrBlock.update (corr.py:157-218): the fused wgmma volume into the tiled pyramid (layout 1) where
        RaftEngine's volume_tiled holds for fmap1 and the modes are 64-channel multiples, else the materialised route (dense, layout 0)."""
        sp = self.corr
        if self.volume_tiled(fmap1, impl) and sp["d"] % 64 == 0:
            q1 = ops.conv2d([ops.layernorm(fmap1, eps=1e-12)], self.corr_qk, torch.empty_like(fmap1), impl=impl)
            k2 = ops.conv2d([ops.layernorm(fmap2t, eps=1e-12)], self.corr_qk, torch.empty_like(fmap2t), impl=impl)
            return ops.craft_volume_tiled(q1, k2, sp["M"], sp["a"], sp["bias"], sp["R"], self.corr_levels), 1
        return self.craft_volume_dense(fmap1, fmap2t, impl), 0

    def craft_volume_dense(self, fmap1: torch.Tensor, fmap2t: torch.Tensor, impl: int = 0) -> List[torch.Tensor]:
        """TransCorrBlock.update (corr.py:157-218): the globally normalised mode mix of LN(fmap1) against LN(fmap2'), and RAFT's
        avg-pool pyramid (dense, layout 0)."""
        B, H, W, _ = fmap1.shape
        sp = self.corr
        scores = self._scores(sp, ops.layernorm(fmap1, eps=1e-12), ops.layernorm(fmap2t, eps=1e-12), impl)
        level = ops.craft_volume_norm(scores, sp["M"], B, H, W, sp["a"], sp["bias"], sp["R"], ops.craft_clamp_flag(scores))
        pyr = [level]
        for _ in range(self.corr_levels - 1):
            q, h, w = pyr[-1].shape
            pyr.append(ops.avg_pool2x2(pyr[-1].view(q, h, w, 1)).view(q, h // 2, w // 2))
        return pyr


# The largest learned diagonal entry an f16 LCV engine takes without a warning.  The volume's values are <f1^T W, f2> / sqrt(C), up to
# max(D) times RAFT's: measured on an H100 with the fnet features of a smooth 436x1024 pair, max |volume| is 71168 at D = 199 (f16
# overflows past 65504) and 22.9k at D = 64, a factor 2.9 below the f16 maximum (DESIGN.md section 5, LCV).
LCV_F16_MAX_D = 64.0


def lcv_bilinear_form(corr_block: torch.nn.Module) -> torch.Tensor:
    """W = P^T D P of LearnableCorrBlock (lcv/corr_lcv.py:19-31) in fp64: S = (triu(raw_P) - triu(raw_P)^T) / 2, P = (I + S)(I - S)^-1
    (Cayley), t = atan(raw_D) 2 / pi, D = diag((1 + t) / (1 - t)).  I is the block's ``eye`` buffer, as the reference reads it."""
    eye = corr_block.eye.detach().double()
    up = torch.triu(corr_block.raw_P.detach().double())
    S = (up - up.t()) / 2
    P = (eye + S) @ torch.inverse(eye - S)
    t = torch.atan(corr_block.raw_D.detach().double()) * 2 / math.pi
    return P.t() @ torch.diag((1 + t) / (1 - t)) @ P


class LCVEngine(RaftEngine):
    """LCV (lcv_raft.py:41-221, corr_lcv.py): RAFT's or raft_small's loop (VARIANT_RAFT / VARIANT_RAFT_SMALL) over the learned volume
    f1^T W f2 / sqrt(C) and a pyramid that stops pooling once a level's smaller side is <= 2r+1.  W / sqrt(C) is folded in fp64 once
    per parameter version (the model keys the engine on the corr_block parameters) and applied to fmap1 as a 1x1 layer; the distinct
    levels are built with scale 1 by the volume builders and the repeated ones alias the last of them (pool_min_side tells the
    lookup their sizes)."""

    def _pack(self, update_block: torch.nn.Module, corr_block: Optional[torch.nn.Module] = None) -> _lib.RaftWeights:
        w = super()._pack(update_block)
        c = corr_block.raw_D.shape[0]
        W = lcv_bilinear_form(corr_block)
        d_max = float(torch.linalg.eigvalsh((W + W.t()) / 2).max())  # max(D): W = P^T D P with P orthogonal
        if self.dtype == torch.float16 and d_max > LCV_F16_MAX_D:
            warnings.warn(f"lcv: the learned diagonal reaches D = {d_max:.0f}, and the f16 correlation volume holds values up to D times "
                          f"RAFT's; above D = {LCV_F16_MAX_D} it can exceed the f16 range (inf in the pyramid, NaN flow). Run this model in "
                          "bfloat16 or float32.", RuntimeWarning, stacklevel=2)
        wf = W / math.sqrt(c)
        # the 1x1 layer's out[j] = sum_i W'[j, i] f1[i] is (f1^T W)[j] for W' = W^T
        self.learned = ops.PackedConv([ConvWeights(wf.t().float()[:, :, None, None].contiguous())], self.dtype, self.device, src_channels=[c])
        self.pool_min_side = 2 * self.corr_radius + 1
        return w

    def _new_workspace(self, cfg: _lib.RaftCfg) -> torch.Tensor:
        # grids whose RAFT pyramid would have an empty level (a 4x4 grid) are valid here
        nbytes = load().pfb_raft_workspace_bytes_ex(C.byref(cfg), self.pool_min_side)
        if nbytes == 0:
            check(-1, "raft_workspace_bytes_ex")
        return torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    def build_volume(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """(the corr_levels levels of compute_cost_volume, of which the repeated ones are the same tensor, its layout)."""
        B, H, W, _ = fmap1.shape
        _, distinct = ops.corr_level_sizes(H, W, self.corr_levels, self.pool_min_side)
        f1w = ops.conv2d([fmap1], self.learned, torch.empty_like(fmap1), impl=impl)
        if self.volume_tiled(fmap1, impl):
            pyr, layout = ops.corr_volume_build_tiled(f1w, fmap2, distinct, scale=1.0), 1
        else:
            pyr, layout = ops.corr_volume_build_ex(f1w, fmap2, distinct, scale=1.0, impl=impl), 0
        return pyr + [pyr[-1]] * (self.corr_levels - distinct), layout


class SplatFlowEngine(RaftEngine):
    """SplatFlow (splatflow.py:86-154, update.py:82-123): GMA's loop (PFB_VARIANT_GMA, one head) run once per frame pair, with two
    weight sets.  ``weights``: the two-frame set, GMA's packing of encoder, gru, flow_head, mask and aggregator (context 128).
    ``three_frame``: the same engine for pair (1, 2) of three frames, whose static GRU input is [inp | mf_t] (context 256): gru_sp with
    its input columns permuted from the reference's [h | inp | mf | mf_s | mf_t] to [h | inp | mf_t | mf | mf_s], so that the loop's
    context split evaluates the inp and mf_t terms once per forward, plus flow_head_sp and mask_sp.  Its encoder and aggregator
    layers are the two-frame set's structs: the shared weights are resident once."""

    def _pack(self, update_block: torch.nn.Module, attention_module: Optional[torch.nn.Module] = None) -> _lib.RaftWeights:
        import copy
        from types import SimpleNamespace

        ub = update_block
        w2 = super()._pack(ub, attention_module)
        layers2 = self.layers
        hd = self.hidden_dim
        perm = torch.cat([torch.arange(2 * hd), torch.arange(4 * hd, 5 * hd), torch.arange(2 * hd, 4 * hd)]).to(ub.gru_sp.convz1.weight.device)

        def permuted(conv):
            return SimpleNamespace(weight=conv.weight.detach()[:, perm].contiguous(), bias=conv.bias, in_channels=conv.in_channels)

        g = ub.gru_sp
        gru_sp = SimpleNamespace(**{n: permuted(getattr(g, n)) for n in ("convz1", "convr1", "convq1", "convz2", "convr2", "convq2")})
        view = SimpleNamespace(encoder=ub.encoder, gru=gru_sp, flow_head=ub.flow_head_sp, mask=ub.mask_sp, aggregator=ub.aggregator)
        three = copy.copy(self)
        three.context_dim = 2 * self.context_dim
        w3 = RaftEngine._pack(three, view, attention_module)
        for k in (_lib.L_CONVC1, _lib.L_CONVC2, _lib.L_CONVF1, _lib.L_CONVF2, _lib.L_CONV, _lib.L_CONVC2F2, _lib.L_AGG_V, _lib.L_AGG_PROJ):
            if k in layers2:
                three.layers[k] = layers2[k]
                w3.layers[k] = w2.layers[k]
            else:
                three.layers.pop(k, None)
        three.weights = w3
        self.three_frame = three
        self.layers = layers2
        return w2

    def motion_features(self, B: int, H: int, W: int, scratch: Optional[dict] = None) -> torch.Tensor:
        """The loop's motion buffer as a pixel-major view [B,H,W,stride] of the workspace that refine(.., scratch) used for this grid:
        channels 0..127 are mf, the motion features of the last iteration (pfb_raft_workspace_motion); read them before the next call
        of the loop on this workspace."""
        cfg = self.make_cfg(B, H, W, 1, (8 * H, 8 * W), (0, 0), False, 0)
        off, stride = C.c_size_t(), C.c_int()
        check(load().pfb_raft_workspace_motion(C.byref(cfg), C.byref(off), C.byref(stride)), "raft_workspace_motion")
        ws = self.workspace(cfg, scratch)
        es = torch.empty((), dtype=self.dtype).element_size()
        n = B * H * W * stride.value * es
        return ws[off.value: off.value + n].view(self.dtype).view(B, H, W, stride.value)
