"""SplatFlow (three-frame motion-feature splatting on the GMA loop) on libptlflow_b200.

Surface kept from ptlflow/models/splatflow/splatflow.py:17-159: class name ``splatflow``, constructor keywords (``corr_levels,
corr_radius, dropout, gamma, max_flow, iters, alternate_corr, fast_inference``), the ``kitti`` checkpoint, state_dict keys (``fnet.*,
cnet.*`` as RAFT's BasicEncoder, ``att.to_qk.weight``, ``update.{encoder, gru, flow_head, mask, aggregator, gru_sp, flow_head_sp,
mask_sp}.*``), ``forward(dict) -> dict`` with ``flows`` and ``flow_small``.  Images are [B, T, 3, H, W], T >= 2:
  * T = 2: pair (0, 1) is GMA's forward with one head and content attention; the model prints a one-time warning, as the reference.
  * T >= 3: pair (0, 1) runs first; its last iteration's motion features mf_01 (the 126 ReLU channels and the 2 flow channels) are
    forward-splatted by its flow (pfb_softsplat_average, "average" mode) into mf_t, which pair (1, 2) reads as a fixed extra GRU
    input (update.gru_sp, flow_head_sp, mask_sp).  The outputs are pair (1, 2)'s.  Frames after the third are never read.
Like the reference, ``corr_levels``, ``corr_radius`` and ``alternate_corr`` are accepted and ignored (always 4 levels of radius 4
over the materialised volume), ``fast_inference`` changes nothing in eval, and ``prev_preds`` is ignored: there is no warm start.

Kernel mapping (DESIGN.md section 1, row a24): fnet runs over frames 0, 1 and 2 as one batch (instance norm is per sample) and cnet
over frames 0 and 1; each pair's volume, attention and loop are GMA's (RaftEngine.refine).  mf_01 is read straight from the loop's
workspace (pfb_raft_workspace_motion) and splatted into the mf_t columns of pair (1, 2)'s static input [inp | mf_t], the loop's
context input of width 256 (ptlflow_b200/engine.py SplatFlowEngine).  The whole forward, both pairs, is one CUDA graph.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn as nn

from ... import ops
from ...engine import SplatFlowEngine
from ...utils.registry import register_model, trainable
from ..gma.gma import GMA, Aggregate
from ..raft.extractor import BasicEncoder
from ..raft.update import BasicMotionEncoder, FlowHead, SepConvGRU, _no_forward


class Attention(nn.Module):
    """attention.py:6-34: content attention only (no position tables), one head of 128 channels."""

    position_only = position_and_content = False

    def __init__(self, *, dim: int, heads: int = 4, dim_head: int = 128) -> None:
        super().__init__()
        self.heads, self.scale = heads, dim_head ** -0.5
        self.to_qk = nn.Conv2d(dim, heads * dim_head * 2, 1, bias=False)

    forward = _no_forward


class Update(nn.Module):
    """update.py:82-107: GMA's update block, plus gru_sp (input [inp | mf | mf_s | mf_t], 640 channels with the hidden state),
    flow_head_sp and mask_sp for the second pair of three frames."""

    def __init__(self, hidden_dim: int = 128) -> None:
        super().__init__()
        self.encoder = BasicMotionEncoder(4, 4)
        self.gru = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim + hidden_dim)
        self.flow_head = FlowHead(hidden_dim, hidden_dim=256)
        self.mask = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1, padding=0))
        self.aggregator = Aggregate(dim=128, dim_head=128, heads=1)
        self.gru_sp = SepConvGRU(hidden_dim=hidden_dim, input_dim=128 + hidden_dim + hidden_dim * 2)
        self.flow_head_sp = FlowHead(hidden_dim, hidden_dim=256)
        self.mask_sp = nn.Sequential(nn.Conv2d(128, 256, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(256, 64 * 9, 1, padding=0))

    forward = _no_forward


class SplatFlow(GMA):
    pretrained_checkpoints = {
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/splatflow-kitti-2aa8e145.ckpt",
    }
    _engine_cls = SplatFlowEngine

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8, max_flow: float = 400,
                 iters: int = 32, alternate_corr: bool = False, fast_inference: bool = True, **kwargs) -> None:
        # the volume is always CorrBlock(fmap1, fmap2, radius=4) with 4 levels (splatflow.py:123, update.py:10-12)
        super().__init__(corr_levels=4, corr_radius=4, dropout=dropout, gamma=gamma, max_flow=max_flow, iters=iters, alternate_corr=False,
                         **kwargs)
        for k, v in (("corr_levels", corr_levels), ("corr_radius", corr_radius), ("alternate_corr", alternate_corr),
                     ("fast_inference", fast_inference)):
            setattr(self.hparams, k, v)  # kept as given, like the reference's attributes; none of them changes the eval forward
        self.fast_inference = fast_inference
        self.has_shown_warning = False

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        self.fnet = BasicEncoder(output_dim=256, norm_fn="instance", dropout=self.dropout)
        self.cnet = BasicEncoder(output_dim=self.hidden_dim + self.context_dim, norm_fn="batch", dropout=self.dropout)
        self.att = Attention(dim=self.context_dim, heads=1, dim_head=self.context_dim)
        self.update = Update(hidden_dim=self.hidden_dim)

    def _engine_module(self) -> nn.Module:
        return self.update

    def _loop_parameters(self):
        return list(self.update.parameters()) + list(self.att.parameters())

    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        images = inputs["images"]
        if images.dim() != 5 or images.shape[1] < 2:
            raise ValueError(f"splatflow needs images [B, T, 3, H, W] with T >= 2 frames; got shape {tuple(images.shape)}")
        if images.shape[1] == 2 and not self.has_shown_warning:
            print("WARNING: splatflow is running in two-frame mode. Provide 3 input images to run in three-frame mode.")
            self.has_shown_warning = True
        # no warm start (splatflow.py:86-118 never reads prev_preds)
        return super().forward({k: v for k, v in inputs.items() if k != "prev_preds"})

    def _forward_device_impl(self, images: torch.Tensor, flow_init, scratch):
        """images [B,T,3,H,W] on the device (only read) -> (flow_up fp32 [B,2,H,W], flow_small fp32 [B,2,H/8,W/8]) of pair (0, 1)
        when T = 2, of pair (1, 2) when T >= 3.  Stream-ordered and free of host synchronisation, like RAFT's (one CUDA graph)."""
        from ...utils.utils import InputPadder

        resizer = InputPadder(images.shape, stride=self.output_stride, pad_mode="replicate", two_side_pad=True)
        B = images.shape[0]
        T = min(images.shape[1], 3)
        frames = ops.preprocess_frames(images, resizer.tgt_size, resizer.pad_top_left, out_channels=self.frame_channels, frames=T)
        # fnet over all T frames in one batch, cnet over the first frame of every pair
        fmap1, fmaps_rest, cnet = self._encode(frames, B, cnet_in=frames[: (T - 1) * B])
        fmaps = [fmap1] + list(fmaps_rest.split(B))
        _, H8, W8, _ = fmap1.shape
        eng = self._get_engine(fmap1.dtype, fmap1.device)
        net, inp = ops.context_split(cnet, self.hidden_dim, self.context_dim)
        attention = self._attention(inp, eng).view(T - 1, B * H8 * W8, H8 * W8)  # one head: the pairs' rows follow each other
        out_hw, pad = tuple(images.shape[-2:]), resizer.pad_top_left

        def run_pair(i: int, engine, static_inp: torch.Tensor):
            coords = ops.init_coords(B, H8, W8, fmap1.device)
            pyramid, layout = engine.build_volume(fmaps[i], fmaps[i + 1], impl=self.kernel_impl)
            return engine.refine(pyramid, layout, net[i * B:(i + 1) * B], static_inp, coords, self.iters, out_hw, pad, attention=attention[i],
                                 scratch=scratch, fork_flow=self.fork_flow)

        flow_up, flow_small = run_pair(0, eng, inp[:B])
        if T == 3:
            # [inp_1 | mf_t]: mf_t = the average splat of mf_01 (still in the loop's workspace) by flow_small_01 (splatflow.py:104-109)
            x2 = torch.empty((B, H8, W8, 2 * self.context_dim), dtype=inp.dtype, device=inp.device)
            x2[..., : self.context_dim] = inp[B:]
            ops.softsplat_average(eng.motion_features(B, H8, W8, scratch), flow_small, out=x2, channels=128, out_offset=self.context_dim)
            flow_up, flow_small = run_pair(1, eng.three_frame, x2)
        return self.postprocess_predictions(flow_up, resizer, is_flow=True), flow_small


@register_model
@trainable
class splatflow(SplatFlow):
    pass
