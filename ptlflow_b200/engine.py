"""RaftEngine: packed weights + workspaces + one C call for the whole refinement loop.

This is the host-side glue between the kept ``RAFT.forward`` structure
(ptlflow/models/raft/raft.py:125-194) and ``pfb_raft_refine``.  It owns nothing numerical:
packing, buffers, pointer structs, CUDA-graph capture.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib, ops
from ._lib import check, dtype_code, load, ptr_array, stream_ptr


_TILED = bool(int(os.environ.get("PFB_VOLUME_TILED", "1")))


class RaftEngine:
    """Built lazily at first forward and rebuilt when the parameters' dtype / device / storage
    change (callers do ``model.eval().cuda().half()`` *after* construction and after
    ``load_state_dict`` -- model_benchmark.py:274-279, infer.py:148-152)."""

    def __init__(self, update_block: torch.nn.Module, variant: int, hidden_dim: int, context_dim: int,
                 corr_levels: int, corr_radius: int, dtype: torch.dtype, device: torch.device, impl: int = 0,
                 attention_module: Optional[torch.nn.Module] = None):
        self.variant, self.hidden_dim, self.context_dim = variant, hidden_dim, context_dim
        self.corr_levels, self.corr_radius = corr_levels, corr_radius
        self.dtype, self.device, self.impl = dtype, device, impl
        ub = update_block
        enc, gru, fh = ub.encoder, ub.gru, ub.flow_head
        planes = corr_levels * (2 * corr_radius + 1) ** 2
        hd, cd = hidden_dim, context_dim

        def P(srcs, *convs):  # srcs: channel counts of the concatenated inputs, in order (wgmma K-major pack)
            return ops.PackedConv(convs, dtype, device, src_channels=srcs)

        layers: Dict[int, ops.PackedConv] = {}
        layers[_lib.L_CONVF1] = P(None, enc.convf1)  # 7x7 on the 2-channel fp32 flow: dedicated kernel
        if variant in (0, 2, 6) and dtype != torch.float32 and tuple(enc.convf1.weight.shape) == (128, 2, 7, 7):
            # tensor-core form (csrc/first_conv.cu): the K-major slot of the layer carries the overlapping-window tiles
            pc = layers[_lib.L_CONVF1]
            pc.weight_k = ops.pack_flow_conv(enc.convf1.weight, dtype).to(device)
            pc.Cin_pad, pc.Cout_pad_k = 64, 128
        if variant in (0, 2, 6):
            layers[_lib.L_CONVC1] = P([planes], enc.convc1)
            layers[_lib.L_CONVC2] = P([256], enc.convc2)
            layers[_lib.L_CONVF2] = P([128], enc.convf2)
            layers[_lib.L_CONV] = P([256], enc.conv)  # cat[cor(192), flo(64)] lives in one 256-channel buffer
            # cat[h or r*h, inp, motion (, motion_global)] -- three tensor maps, no concat copy (gma keeps
            # motion | motion_global in one 256-channel buffer, and so does ccmr)
            gsrc = [hd, cd, 256 if variant in (2, 6) else 128]
            layers[_lib.L_GRU_ZR1] = P(gsrc, gru.convz1, gru.convr1)  # z | r share the input: one GEMM, N = 2*hidden
            layers[_lib.L_GRU_Q1] = P(gsrc, gru.convq1)
            layers[_lib.L_GRU_ZR2] = P(gsrc, gru.convz2, gru.convr2)
            layers[_lib.L_GRU_Q2] = P(gsrc, gru.convq2)
            if dtype != torch.float32:
                # round 2: (a) the context columns of the four GRU convolutions become layers of their own, evaluated once per
                # forward with the bias folded in, and the per-iteration layers lose them (-1/3 of the GRU's K); (b) convc2 |
                # convf2 as one block-diagonal N = 256 layer.  Pure repacking of the same parameters.
                class _View:
                    def __init__(self, weight, bias):
                        self.weight, self.bias = weight, bias

                def cols(conv, lo, hi, with_bias):
                    return _View(conv.weight.detach()[:, lo:hi].contiguous(), conv.bias if with_bias else None)

                def rest(conv):  # [h | inp | motion...] without the inp columns
                    w = conv.weight.detach()
                    return _View(torch.cat([w[:, :hd], w[:, hd + cd:]], dim=1).contiguous(), None)

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
                    layers[_lib.L_CONVC2F2] = P([wc.shape[1], wf.shape[1]], _View(bd, torch.cat([enc.convc2.bias.detach(), enc.convf2.bias.detach()])))
            layers[_lib.L_FLOW1] = P([hd], fh.conv1)
            layers[_lib.L_FLOW2] = P([256], fh.conv2)
            if dtype != torch.float32:
                # conv2 as a 1x1 layer producing the 9 x 2 per-tap products (row = tap*2 + o); bias is added by the gather
                class _Taps:
                    def __init__(self, w):
                        self.weight, self.bias = w.detach().permute(2, 3, 0, 1).reshape(18, w.shape[1], 1, 1).contiguous(), None

                layers[_lib.L_FLOW2T] = P([256], _Taps(fh.conv2.weight))
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
        self.agg_gamma = 0.0
        self.num_heads = 1
        self.att_q = self.att_k = self.att_pos = None
        if variant == 2:
            layers[_lib.L_AGG_V], proj = self._pack_attention(ub.aggregator, attention_module)
            if proj is not None:
                layers[_lib.L_AGG_PROJ] = proj
        self.layers = layers
        self.weights = _lib.RaftWeights()
        for k, v in layers.items():
            self.weights.layers[k] = v.layer_struct()
        self._workspaces: Dict[Tuple, torch.Tensor] = {}
        self.signature = self.param_signature(update_block)
        # the pack kernels ran on the constructing thread's stream; other streams / host threads (pipeline slots) may use
        # the packed weights as soon as the engine is published, so finish them first (one-time cost)
        torch.cuda.current_stream(device).synchronize()

    def _pack_attention(self, agg: torch.nn.Module, attention_module: torch.nn.Module):
        """GMA's Aggregate and Attention (gma_utils.py:32-113): sets num_heads, agg_gamma and the per-head q / k / position layers
        of the attention; returns the packed (to_v, project or None) of the per-iteration aggregate."""
        dtype, device = self.dtype, self.device
        self.num_heads = agg.heads
        to_v = ops.PackedConv([agg.to_v], dtype, device, src_channels=[128])
        proj = ops.PackedConv([agg.project], dtype, device, src_channels=[agg.project.weight.shape[1]]) if agg.project is not None else None
        self.agg_gamma = float(agg.gamma.detach().float().cpu().item())

        class _Half:  # one head's q / k block of Attention.to_qk as a 1x1 layer (contiguous head-major outputs for the GEMM)
            def __init__(self, w):
                self.weight, self.bias = w, None

        wqk = attention_module.to_qk.weight
        c = wqk.shape[0] // 2
        d = c // self.num_heads  # dim_head
        cin = [wqk.shape[1]]
        self.att_q = [ops.PackedConv([_Half(wqk[h * d:(h + 1) * d])], dtype, device, src_channels=cin) for h in range(self.num_heads)]
        self.att_k = [ops.PackedConv([_Half(wqk[c + h * d:c + (h + 1) * d])], dtype, device, src_channels=cin)
                      for h in range(self.num_heads)]
        if attention_module.position_only or attention_module.position_and_content:
            # per-query position tables of head h: scale * q_h . [rel_height; rel_width] (gma_utils.py:18-30) = a 1x1 layer on
            # `inp` whose weight is [E_h; E_w] @ W_q,h ((2P-1) * 2 rows, folded in fp64), scale applied by the epilogue
            pe = attention_module.pos_emb
            emb = torch.cat([pe.rel_height.weight, pe.rel_width.weight], 0).detach().double()
            self.att_pos = [ops.PackedConv([_Half((emb @ wqk[h * d:(h + 1) * d, :, 0, 0].detach().double()).float()[:, :, None, None])],
                                           dtype, device, src_channels=cin) for h in range(self.num_heads)]
            self.max_pos = pe.rel_height.weight.shape[0] // 2 + 1
        return to_v, proj

    # -- cache invalidation --------------------------------------------------------------------
    @staticmethod
    def param_signature(update_block: torch.nn.Module):
        return tuple((p.data_ptr(), p._version, p.dtype, str(p.device)) for p in update_block.parameters())

    # -- run --------------------------------------------------------------------------------
    def make_cfg(self, B: int, H: int, W: int, iters: int, out_hw, pad, alternate_corr: bool, feat_dim: int, volume_layout: int = 0) -> _lib.RaftCfg:
        return _lib.RaftCfg(self.variant, dtype_code(self.dtype), B, H, W, feat_dim, self.corr_levels, self.corr_radius,
                            self.hidden_dim, self.context_dim, iters, int(alternate_corr), out_hw[0], out_hw[1], pad[0], pad[1],
                            self.impl, 0 if alternate_corr else int(volume_layout), int(getattr(self, "fork_flow", False)), self.num_heads)

    def build_volume(self, fmap1: torch.Tensor, fmap2: torch.Tensor, impl: int = 0):
        """a1 + a2 for the refinement loop of this engine.  f16 / bf16 with tensor-core-shaped features get the tiled
        pyramid (64-byte tiles, csrc/corr_tiled.cu); everything else the dense one.  refine() reads the layout back from
        ``self.volume_layout`` (set here, per call)."""
        self.volume_layout = 0
        if _TILED and impl != 1 and self.corr_radius in (3, 4) and ops.tiled_supported(fmap1, self.corr_levels) \
                and (self.corr_radius, self.corr_levels) in ((4, 4), (4, 3), (4, 2), (4, 1), (3, 4), (3, 3)):
            self.volume_layout = 1
            return ops.corr_volume_build_tiled(fmap1, fmap2, self.corr_levels)
        return ops.corr_volume_build(fmap1, fmap2, self.corr_levels, impl=impl)

    # C entry points of this engine's loop (SKFlowEngine runs its own with the same cfg / buffers)
    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_raft_workspace_bytes", "pfb_raft_refine", "pfb_raft_update_iter"

    def workspace(self, cfg: _lib.RaftCfg, scratch: Optional[dict] = None) -> torch.Tensor:
        if scratch is not None:
            # the caller owns the scratch memory (a CUDA graph keeps the workspace it was captured with alive)
            key = ("raft_ws", cfg.B, cfg.H, cfg.W)
            ws = scratch.get(key)
            if ws is None:
                nbytes = getattr(load(), self._ws_symbol)(C.byref(cfg))
                if nbytes == 0:
                    check(-1, "raft_workspace_bytes")
                ws = scratch[key] = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            return ws
        # one workspace per CUDA stream (batches in flight on different streams must not share scratch memory,
        # ptlflow_b200/pipeline.py) and, per stream, one shape resident (bounded memory, SURVEY appendix B.7)
        sid = torch.cuda.current_stream(self.device).cuda_stream
        key = (cfg.B, cfg.H, cfg.W)
        ent = self._workspaces.get(sid)
        if ent is None or ent[0] != key:
            nbytes = getattr(load(), self._ws_symbol)(C.byref(cfg))
            if nbytes == 0:
                check(-1, "raft_workspace_bytes")
            ent = (key, torch.empty(nbytes, dtype=torch.uint8, device=self.device))
            if len(self._workspaces) >= 8:
                # streams come and go: do not grow without bound.  A dropped tensor returns to torch's caching allocator,
                # which keeps the block reserved for the stream it was allocated on until that stream's queued work is
                # done -- an evicted workspace with work still in flight is therefore not reused under that work.
                self._workspaces.pop(next(iter(self._workspaces)))
            self._workspaces[sid] = ent
        return ent[1]

    def refine(self, pyramid: Sequence[torch.Tensor], net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor,
               iters: int, out_hw, pad, fmap1: Optional[torch.Tensor] = None, attention: Optional[torch.Tensor] = None,
               scratch: Optional[dict] = None):
        """Runs the loop in place on (net, coords); returns (flow_up fp32 [B,2,oh,ow], flow_small fp32 [B,2,H,W])."""
        B, H, W, _ = net.shape
        alt = fmap1 is not None
        cfg = self.make_cfg(B, H, W, iters, out_hw, pad, alt, fmap1.shape[-1] if alt else 0, getattr(self, "volume_layout", 0))
        ws = self.workspace(cfg, scratch)
        flow_up = torch.empty((B, 2, out_hw[0], out_hw[1]), dtype=torch.float32, device=self.device)
        flow_small = torch.empty((B, 2, H, W), dtype=torch.float32, device=self.device)
        pyr = ptr_array(pyramid)
        buf = _lib.RaftBuffers(C.cast(pyr, C.POINTER(C.c_void_p)), fmap1.data_ptr() if alt else None, net.data_ptr(),
                               inp.data_ptr(), coords.data_ptr(), flow_up.data_ptr(), flow_small.data_ptr(),
                               ws.data_ptr(), ws.numel(), attention.data_ptr() if attention is not None else None, self.agg_gamma)
        with torch.cuda.device(self.device):
            check(getattr(load(), self._refine_symbol)(C.byref(cfg), C.byref(self.weights), C.byref(buf), stream_ptr(self.device)),
                  self._refine_symbol[4:])
        return flow_up, flow_small

    def update_iter(self, net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, corr: Optional[torch.Tensor] = None,
                    pyramid: Optional[Sequence[torch.Tensor]] = None, want_mask: bool = False, attention: Optional[torch.Tensor] = None):
        """One update-block evaluation (operator-level tests).  corr: pixel-major [B,H,W,planes]; attention (gma): head-major
        [heads*B*N, N]."""
        B, H, W, _ = net.shape
        cfg = self.make_cfg(B, H, W, 1, (8 * H, 8 * W), (0, 0), False, 0)
        ws = self.workspace(cfg)
        mask = torch.empty((B, H, W, 576), dtype=self.dtype, device=self.device) if (want_mask and self.variant in (0, 3, 4)) else None
        pyr = ptr_array(pyramid) if pyramid is not None else None
        buf = _lib.RaftBuffers(C.cast(pyr, C.POINTER(C.c_void_p)) if pyr is not None else None, None, net.data_ptr(), inp.data_ptr(),
                               coords.data_ptr(), None, None, ws.data_ptr(), ws.numel(),
                               attention.data_ptr() if attention is not None else None, self.agg_gamma)
        with torch.cuda.device(self.device):
            check(getattr(load(), self._iter_symbol)(C.byref(cfg), C.byref(self.weights), C.byref(buf),
                                                     corr.data_ptr() if corr is not None else None,
                                                     mask.data_ptr() if mask is not None else None, stream_ptr(self.device)),
                  self._iter_symbol[4:])
        return mask


def _align(n: int, a: int) -> int:
    return (n + a - 1) // a * a


class _View:
    """weight / bias pair shaped like an nn.Conv2d, for PackedConv."""

    def __init__(self, weight, bias):
        self.weight, self.bias = weight, bias


def _pad_conv(conv: torch.nn.Module, cout: int, cin: int) -> _View:
    """conv's weight / bias zero-padded to [cout, cin, kh, kw] / [cout]."""
    w = conv.weight.detach()
    wp = torch.zeros((cout, cin) + tuple(w.shape[2:]), dtype=w.dtype, device=w.device)
    wp[: w.shape[0], : w.shape[1]] = w
    b = None
    if conv.bias is not None:
        b = torch.zeros(cout, dtype=conv.bias.dtype, device=conv.bias.device)
        b[: conv.bias.shape[0]] = conv.bias.detach()
    return _View(wp, b)


class SKFlowEngine(RaftEngine):
    """SKFlow's update block (skflow/update.py:7-99) packed for pfb_skflow_refine: every PCBlock's 1x1 layers through
    ops.PackedConv, its depthwise filters as fp32 [k*k][C], all channel counts zero-padded to multiples of 32 (the padding stays
    exactly zero through the block).  Same lifecycle and invalidation as RaftEngine; the attention is GMA's."""

    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_skflow_workspace_bytes", "pfb_skflow_refine", "pfb_skflow_update_iter"

    def __init__(self, update_block: torch.nn.Module, variant: int, hidden_dim: int, context_dim: int,
                 corr_levels: int, corr_radius: int, dtype: torch.dtype, device: torch.device, impl: int = 0,
                 attention_module: Optional[torch.nn.Module] = None):
        self.variant, self.hidden_dim, self.context_dim = variant, hidden_dim, context_dim
        self.corr_levels, self.corr_radius = corr_levels, corr_radius
        self.dtype, self.device, self.impl = dtype, device, impl
        ub = update_block
        enc = ub.encoder
        planes = corr_levels * (2 * corr_radius + 1) ** 2
        self._keep: List[object] = []  # everything the weight struct points into
        w = _lib.SkflowWeights()
        blocks = ((_lib.SK_CONVC1, enc.convc1, planes), (_lib.SK_CONVC2, enc.convc2, 256), (_lib.SK_CONVF2, enc.convf2, 128),
                  (_lib.SK_CONV, enc.conv, 256), (_lib.SK_GRU, ub.gru, 512), (_lib.SK_FLOW_HEAD, ub.flow_head, 128))
        for bid, blk, cin in blocks:
            w.blocks[bid] = self._pack_block(blk, cin)
        self.corr_stride = _align(planes, 32)  # the lookup buffer: planes channels, zero up to the padded width
        for name, conv, srcs in (("convf1", enc.convf1, None), ("mask1", ub.mask[0], [128]), ("mask2", ub.mask[2], [256])):
            setattr(w, name, self._layer(ops.PackedConv([conv], dtype, device, src_channels=srcs)))
        to_v, proj = self._pack_attention(ub.aggregator, attention_module)
        w.agg_v = self._layer(to_v)
        if proj is not None:
            w.agg_proj = self._layer(proj)
        self.weights = w
        self._workspaces: Dict[Tuple, torch.Tensor] = {}
        self.signature = self.param_signature(update_block)
        torch.cuda.current_stream(device).synchronize()

    def _layer(self, pc: ops.PackedConv) -> _lib.Layer:
        self._keep.append(pc)
        return pc.layer_struct()

    def _pack_block(self, blk: torch.nn.Module, cin: int) -> _lib.PcBlock:
        """PCBlock4_Deep_nopool_res(cin, cout, k_conv) -> pfb_pc_block (C = align(cin, 32), hid = align(int(1.5 cin), 32))."""
        dtype, device = self.dtype, self.device
        C, hid = _align(cin, 32), _align(int(1.5 * cin), 32)
        cout = blk.ffn2[2].weight.shape[0]

        def P(view, srcs):
            return self._layer(ops.PackedConv([view], dtype, device, src_channels=srcs))

        k = _lib.PcBlock()
        k.ffn1a = P(_pad_conv(blk.ffn1[0], hid, C), [C])
        k.ffn1b = P(_pad_conv(blk.ffn1[2], C, hid), [hid])
        k.pw = P(_pad_conv(blk.pw, C, C), [C])
        k.ffn2a = P(_pad_conv(blk.ffn2[0], hid, C), [C])
        k.ffn2b = P(_pad_conv(blk.ffn2[2], cout, hid), [hid])
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


def _searaft_params(model: torch.nn.Module):
    """The parameters SEARaftEngine packs: init_conv, the heads and (iters > 0) the update block."""
    mods = [model.init_conv, model.flow_head, model.upsample_weight] + ([model.update_block] if hasattr(model, "update_block") else [])
    return [p for m in mods for p in m.parameters()]


class SEARaftEngine(RaftEngine):
    """SEA-RAFT's heads and update block (sea_raft.py:104-133, update.py:18-54, layer.py:41-83) packed for pfb_searaft_refine.  Each
    ConvNextBlock becomes its depthwise filter (fp32 [k*k][384]) and two 1x1 layers, folded in fp64 from the parameters:
    pw1 = pwconv1 with the LayerNorm affine (W1 diag(ln_w), b1 + W1 ln_b), and out = final(x + gamma * pwconv2(h)) over the two
    sources [h | x] ([Wf diag(gamma) W2 | Wf], Wf (gamma b2) + bf).  Same lifecycle and invalidation as RaftEngine, keyed on
    every parameter it packs."""

    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_searaft_workspace_bytes", "pfb_searaft_refine", "pfb_searaft_update_iter"

    @staticmethod
    def param_signature(model: torch.nn.Module):
        return tuple((p.data_ptr(), p._version, p.dtype, str(p.device)) for p in _searaft_params(model))

    def __init__(self, model: torch.nn.Module, variant: int, hidden_dim: int, context_dim: int, corr_levels: int, corr_radius: int,
                 dtype: torch.dtype, device: torch.device, impl: int = 0):
        self.variant, self.hidden_dim, self.context_dim = variant, hidden_dim, context_dim
        self.corr_levels, self.corr_radius = corr_levels, corr_radius
        self.dtype, self.device, self.impl = dtype, device, impl
        self.agg_gamma, self.num_heads = 0.0, 1
        self._keep: List[object] = []  # everything the weight struct points into
        w = _lib.SearaftWeights()

        def P(conv, srcs):
            return self._layer(ops.PackedConv([conv], dtype, device, src_channels=srcs))

        w.init_conv = P(model.init_conv, [256])
        fh = model.flow_head
        w.flow1 = P(fh[0], [128])
        w2, b2 = fh[2].weight.detach()[:2], fh[2].bias.detach()[:2]  # the flow outputs; info (2:6) feeds training only
        w.flow2 = P(_View(w2.contiguous(), b2.contiguous()), [256])
        if dtype != torch.float32:  # 3x3 -> 2 as a 1x1 layer to the 9 x 2 per-tap products (row = tap*2 + o); the gather adds the bias
            w.flow2t = P(_View(w2.permute(2, 3, 0, 1).reshape(18, w2.shape[1], 1, 1).contiguous(), None), [256])
        w.mask1 = P(model.upsample_weight[0], [128])
        w.mask2 = P(model.upsample_weight[2], [256])
        w.ln_eps = 1e-6
        ub = getattr(model, "update_block", None)
        if ub is not None:
            enc = ub.encoder
            planes = corr_levels * (2 * corr_radius + 1) ** 2
            w.convc1, w.convc2 = P(enc.convc1, [planes]), P(enc.convc2, [256])
            w.convf1 = P(enc.convf1, None)
            if dtype != torch.float32 and tuple(enc.convf1.weight.shape) == (128, 2, 7, 7):
                pc = self._keep[-1]  # tensor-core form (csrc/first_conv.cu): the K-major slot carries the overlapping-window tiles
                pc.weight_k = ops.pack_flow_conv(enc.convf1.weight, dtype).to(device)
                pc.Cin_pad, pc.Cout_pad_k = 64, 128
                w.convf1 = pc.layer_struct()
            w.convf2, w.conv = P(enc.convf2, [128]), P(enc.conv, [256])
            if len(ub.refine) > _lib.PFB_SR_MAX_BLOCKS:
                raise ValueError(f"sea_raft: at most {_lib.PFB_SR_MAX_BLOCKS} ConvNeXt blocks, got {len(ub.refine)}")
            w.num_blocks = len(ub.refine)
            for i, blk in enumerate(ub.refine):
                w.blocks[i] = self._pack_block(blk)
                w.ln_eps = blk.norm.eps
        self.weights = w
        self._workspaces: Dict[Tuple, torch.Tensor] = {}
        self.signature = self.param_signature(model)
        torch.cuda.current_stream(device).synchronize()

    def _layer(self, pc: ops.PackedConv) -> _lib.Layer:
        self._keep.append(pc)
        return pc.layer_struct()

    def _pack_block(self, blk: torch.nn.Module) -> _lib.ConvNextBlock:
        dtype, device = self.dtype, self.device
        f64 = lambda t: t.detach().to(device, torch.float64)  # noqa: E731
        W1, b1, lw, lb = f64(blk.pwconv1.weight), f64(blk.pwconv1.bias), f64(blk.norm.weight), f64(blk.norm.bias)
        W2, b2, g = f64(blk.pwconv2.weight), f64(blk.pwconv2.bias), f64(blk.gamma)
        Wf, bf = f64(blk.final.weight)[:, :, 0, 0], f64(blk.final.bias)
        pw1 = _View((W1 * lw[None, :]).float()[:, :, None, None].contiguous(), (b1 + W1 @ lb).float())
        out = _View(torch.cat([Wf @ (g[:, None] * W2), Wf], 1).float()[:, :, None, None].contiguous(), (Wf @ (g * b2) + bf).float())
        C, k = blk.dwconv.weight.shape[0], blk.dwconv.weight.shape[-1]
        dw_w = blk.dwconv.weight.detach().to(device, torch.float32).reshape(C, k * k).t().contiguous()  # [tap][channel]
        dw_b = blk.dwconv.bias.detach().to(device, torch.float32).contiguous()
        self._keep += [dw_w, dw_b]
        b = _lib.ConvNextBlock()
        b.dw_k, b.dw_weight, b.dw_bias = k, dw_w.data_ptr(), dw_b.data_ptr()
        b.pw1 = self._layer(ops.PackedConv([pw1], dtype, device, src_channels=[C]))
        b.out = self._layer(ops.PackedConv([out], dtype, device, src_channels=[4 * Wf.shape[0], C]))
        return b


class MSRaftEngine(RaftEngine):
    """MS-RAFT+'s update block (ms_raft_plus/update.py:119-153: RAFT's BasicUpdateBlock with convc1 over levels * (2r+1)^2 planes and
    a 36-channel mask head) packed exactly as RaftEngine packs raft's, driven one scale at a time through pfb_msraft_refine
    (pfb_raft_cfg variant 5)."""

    _ws_symbol, _refine_symbol, _iter_symbol = "pfb_msraft_workspace_bytes", "pfb_msraft_refine", "pfb_msraft_update_iter"

    def __init__(self, update_block: torch.nn.Module, variant: int, hidden_dim: int, context_dim: int, corr_levels: int, corr_radius: int,
                 dtype: torch.dtype, device: torch.device, impl: int = 0, attention_module: Optional[torch.nn.Module] = None):
        super().__init__(update_block, 0, hidden_dim, context_dim, corr_levels, corr_radius, dtype, device, impl=impl)  # raft's packing
        self.variant = variant

    def refine_scale(self, pyramid: Sequence[torch.Tensor], net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, iters: int,
                     out_hw, pad, ws: torch.Tensor, fmap1: Optional[torch.Tensor] = None, corr_scale: float = 0.0,
                     volume_layout: int = 0, last: bool = False):
        """One scale in place on (net, coords).  Not last: returns the next scale's coordinates fp32 [B,2H,2W,2].  Last: returns
        (flow_up fp32 [B,2,oh,ow], flow_small fp32 [B,2,oh//16,ow//16])."""
        B, H, W, _ = net.shape
        alt = fmap1 is not None
        cfg = self.make_cfg(B, H, W, iters, out_hw, pad, alt, fmap1.shape[-1] if alt else 0, volume_layout)
        flow_up = flow_small = nxt = None
        if last:
            flow_up = torch.empty((B, 2, out_hw[0], out_hw[1]), dtype=torch.float32, device=self.device)
            flow_small = torch.empty((B, 2, out_hw[0] // 16, out_hw[1] // 16), dtype=torch.float32, device=self.device)
        else:
            nxt = torch.empty((B, 2 * H, 2 * W, 2), dtype=torch.float32, device=self.device)
        pyr = ptr_array(pyramid)
        buf = _lib.RaftBuffers(C.cast(pyr, C.POINTER(C.c_void_p)), fmap1.data_ptr() if alt else None, net.data_ptr(), inp.data_ptr(),
                               coords.data_ptr(), flow_up.data_ptr() if last else None, flow_small.data_ptr() if last else None,
                               ws.data_ptr(), ws.numel(), None, 0.0)
        with torch.cuda.device(self.device):
            check(load().pfb_msraft_refine(C.byref(cfg), C.byref(self.weights), C.byref(buf), corr_scale,
                                           nxt.data_ptr() if nxt is not None else None, stream_ptr(self.device)), "msraft_refine")
        return (flow_up, flow_small) if last else nxt

    def update_iter(self, net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, corr: Optional[torch.Tensor] = None,
                    pyramid: Optional[Sequence[torch.Tensor]] = None, want_mask: bool = False, attention: Optional[torch.Tensor] = None,
                    fmap1: Optional[torch.Tensor] = None, corr_scale: float = 0.0):
        """One update-block evaluation (operator-level tests); returns the [B,H,W,36] mask when asked."""
        B, H, W, _ = net.shape
        alt = fmap1 is not None
        cfg = self.make_cfg(B, H, W, 1, (2 * H, 2 * W), (0, 0), alt, fmap1.shape[-1] if alt else 0)
        ws = self.workspace(cfg)
        mask = torch.empty((B, H, W, 36), dtype=self.dtype, device=self.device) if want_mask else None
        pyr = ptr_array(pyramid) if pyramid is not None else None
        buf = _lib.RaftBuffers(C.cast(pyr, C.POINTER(C.c_void_p)) if pyr is not None else None, fmap1.data_ptr() if alt else None,
                               net.data_ptr(), inp.data_ptr(), coords.data_ptr(), None, None, ws.data_ptr(), ws.numel(), None, 0.0)
        with torch.cuda.device(self.device):
            check(load().pfb_msraft_update_iter(C.byref(cfg), C.byref(self.weights), C.byref(buf),
                                                corr.data_ptr() if corr is not None else None,
                                                mask.data_ptr() if mask is not None else None, corr_scale, stream_ptr(self.device)),
                  "msraft_update_iter")
        return mask


class CCMREngine(RaftEngine):
    """CCMR's update block (ccmr/update.py:110-168: MS-RAFT+'s layers with a GMA-width GRU over [inp | motion | motion_global]) packed
    as RaftEngine packs gma's, plus per scale the XCiT of the context (``xcit[i]``) and the aggregator (``update_block.aggregator[i]``)
    as pfb_xcit_block descriptors, folded in fp64 (xcit.py:242-300): norm1's affine into q | k and v, gamma1 into proj, gamma3 into
    LPI's second convolution, norm2's affine into fc1 and gamma2 into fc2.  Driven one scale at a time through pfb_ccmr_refine
    (pfb_raft_cfg variant 6)."""

    def __init__(self, update_block: torch.nn.Module, variant: int, hidden_dim: int, context_dim: int, corr_levels: int, corr_radius: int,
                 dtype: torch.dtype, device: torch.device, impl: int = 0, xcit: Optional[torch.nn.Module] = None):
        super().__init__(update_block, variant, hidden_dim, context_dim, corr_levels, corr_radius, dtype, device, impl=impl)
        self._keep: List[object] = []
        self.scale_weights = []
        for i in range(len(update_block.aggregator)):
            w = _lib.CcmrWeights()
            w.raft = self.weights
            w.context = self._pack_xcit(xcit[i], separate=False)
            w.aggregator = self._pack_xcit(update_block.aggregator[i], separate=True)
            self.scale_weights.append(w)
        torch.cuda.current_stream(device).synchronize()

    def _pack_xcit(self, xc: torch.nn.Module, separate: bool) -> _lib.XcitBlock:
        dtype, device = self.dtype, self.device
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

        def P(weight, bias, cin):
            pc = ops.PackedConv([_View(weight.float()[:, :, None, None].contiguous(), bias.float().contiguous())], dtype, device,
                                src_channels=[cin])
            self._keep.append(pc)
            return pc.layer_struct()

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

    _ws_symbol = "pfb_ccmr_workspace_bytes"

    def refine_scale(self, scale: int, pyramid: Sequence[torch.Tensor], net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, iters: int,
                     out_hw, pad, ws: torch.Tensor, fmap1: Optional[torch.Tensor] = None, corr_scale: float = 0.0, volume_layout: int = 0,
                     last: bool = False, upflow2: int = 0):
        """One scale in place on (net, coords).  Not last: returns the next scale's coordinates fp32 [B,2H,2W,2].  Last: returns
        (flow_up fp32 [B,2,oh,ow], flow_small fp32 [B,2,oh//16,ow//16])."""
        B, H, W, _ = net.shape
        alt = fmap1 is not None
        cfg = self.make_cfg(B, H, W, iters, out_hw, pad, alt, fmap1.shape[-1] if alt else 0, volume_layout)
        flow_up = flow_small = nxt = None
        if last:
            flow_up = torch.empty((B, 2, out_hw[0], out_hw[1]), dtype=torch.float32, device=self.device)
            flow_small = torch.empty((B, 2, out_hw[0] // 16, out_hw[1] // 16), dtype=torch.float32, device=self.device)
        else:
            nxt = torch.empty((B, 2 * H, 2 * W, 2), dtype=torch.float32, device=self.device)
        pyr = ptr_array(pyramid)
        buf = _lib.RaftBuffers(C.cast(pyr, C.POINTER(C.c_void_p)), fmap1.data_ptr() if alt else None, net.data_ptr(), inp.data_ptr(),
                               coords.data_ptr(), flow_up.data_ptr() if last else None, flow_small.data_ptr() if last else None,
                               ws.data_ptr(), ws.numel(), None, 0.0)
        with torch.cuda.device(self.device):
            check(load().pfb_ccmr_refine(C.byref(cfg), C.byref(self.scale_weights[scale]), C.byref(buf), corr_scale, int(upflow2),
                                         nxt.data_ptr() if nxt is not None else None, stream_ptr(self.device)), "ccmr_refine")
        return (flow_up, flow_small) if last else nxt

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

    def update_iter(self, net: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, corr: Optional[torch.Tensor] = None,
                    pyramid: Optional[Sequence[torch.Tensor]] = None, want_mask: bool = False, attention: Optional[torch.Tensor] = None,
                    fmap1: Optional[torch.Tensor] = None, corr_scale: float = 0.0, scale: int = 0):
        """One update-block evaluation of scale ``scale`` (operator-level tests); returns the [B,H,W,36] mask when asked."""
        B, H, W, _ = net.shape
        alt = fmap1 is not None
        cfg = self.make_cfg(B, H, W, 1, (2 * H, 2 * W), (0, 0), alt, fmap1.shape[-1] if alt else 0)
        ws = self.workspace(cfg)
        mask = torch.empty((B, H, W, 36), dtype=self.dtype, device=self.device) if want_mask else None
        pyr = ptr_array(pyramid) if pyramid is not None else None
        buf = _lib.RaftBuffers(C.cast(pyr, C.POINTER(C.c_void_p)) if pyr is not None else None, fmap1.data_ptr() if alt else None,
                               net.data_ptr(), inp.data_ptr(), coords.data_ptr(), None, None, ws.data_ptr(), ws.numel(), None, 0.0)
        with torch.cuda.device(self.device):
            check(load().pfb_ccmr_update_iter(C.byref(cfg), C.byref(self.scale_weights[scale]), C.byref(buf),
                                              corr.data_ptr() if corr is not None else None, mask.data_ptr() if mask is not None else None,
                                              corr_scale, stream_ptr(self.device)), "ccmr_update_iter")
        return mask
