"""RAFT / RAFTSmall behind the reference's model surface, running on libptlflow_b200.

Kept from the reference (ptlflow/models/raft/raft.py:48-247): class names, constructor keywords
(= hparams / CLI flags), ``state_dict`` keys, ``forward(inputs: dict) -> dict`` with ``flows``
[B,1,2,H,W] and ``flow_small`` [B,2,H/8,W/8], the warm-start input ``prev_preds.flow_small``.
Replaced: everything between the encoders and the returned flow -- correlation volume + pyramid,
the ``iters`` x {lookup, motion encoder, (Sep)ConvGRU, flow head}, mask head and the convex
upsample run as hand-written sm_90a kernels through one C call (ptlflow_b200/engine.py).
"""
from __future__ import annotations

from typing import Dict, Optional

import contextlib
import threading

import torch
import torch.nn as nn

from ... import _lib, ops
from ...engine import RaftEngine
from ...utils.registry import ptlflow_trained, register_model, trainable
from ..base_model.base_model import BaseModel
from .extractor import BasicEncoder, SmallEncoder
from .update import BasicUpdateBlock, SmallUpdateBlock


class _CaptureGate:
    """Readers-writer gate between forwards and CUDA-graph captures of this process: any number of forwards (eager or
    replayed) run together, a capture runs alone.  Host threads that launch and allocate while another thread's stream
    is capturing (pipeline slots on their first batches) made the capture, or their own calls, fail with
    ``cudaErrorStreamCaptureUnsupported`` now and then; captures are rare (once per shape and stream), so excluding them
    costs nothing in steady state."""

    def __init__(self) -> None:
        self._cond = threading.Condition()
        self._readers = 0
        self._writer = False
        self._writers_waiting = 0

    @contextlib.contextmanager
    def forward(self):
        if not _GATE_FORWARDS:
            yield
            return
        with self._cond:
            while self._writer or self._writers_waiting:
                self._cond.wait()
            self._readers += 1
        try:
            yield
        finally:
            with self._cond:
                self._readers -= 1
                if self._readers == 0:
                    self._cond.notify_all()

    @contextlib.contextmanager
    def capture(self):
        with self._cond:
            self._writers_waiting += 1
            while self._writer or self._readers:
                self._cond.wait()
            self._writers_waiting -= 1
            self._writer = True
        try:
            yield
        finally:
            with self._cond:
                self._writer = False
                self._cond.notify_all()


_gate = _CaptureGate()  # one CUDA-graph capture at a time per process, and no forward of another host thread beside it
_GATE_FORWARDS = bool(int(__import__("os").environ.get("PFB_CAPTURE_EXCLUSIVE", "1")))
_cudnn_lock = threading.Lock()
_cudnn_users = 0
_cudnn_saved = None


@contextlib.contextmanager
def _cudnn_flags(benchmark: bool, allow_tf32: bool):
    """torch.backends.cudnn.flags() saves / restores process-global flags; with several forwards in flight on
    different host threads (pipeline.FramePipeline) the first to leave would switch benchmark mode off under the
    others.  First in sets, last out restores."""
    global _cudnn_users, _cudnn_saved
    cd = torch.backends.cudnn
    with _cudnn_lock:
        if _cudnn_users == 0:
            _cudnn_saved = (cd.enabled, cd.benchmark, cd.allow_tf32)
            cd.enabled, cd.benchmark, cd.allow_tf32 = True, benchmark, allow_tf32
        _cudnn_users += 1
    try:
        yield
    finally:
        with _cudnn_lock:
            _cudnn_users -= 1
            if _cudnn_users == 0:
                cd.enabled, cd.benchmark, cd.allow_tf32 = _cudnn_saved


class SequenceLoss(nn.Module):
    """Exponentially weighted L1 over the prediction sequence (training only; kept because the
    constructor stores it as ``loss_fn``)."""

    def __init__(self, gamma: float, max_flow: float) -> None:
        super().__init__()
        self.gamma, self.max_flow = gamma, max_flow

    def forward(self, outputs, inputs):
        preds = outputs["flow_preds"]
        gt, valid = inputs["flows"][:, 0], inputs["valids"][:, 0]
        valid = (valid >= 0.5) & (gt.pow(2).sum(dim=1, keepdim=True).sqrt() < self.max_flow)
        n = len(preds)
        return sum(self.gamma ** (n - i - 1) * (valid * (p - gt).abs()).mean() for i, p in enumerate(preds))


class RAFT(BaseModel):
    pretrained_checkpoints = {
        "chairs": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/raft-chairs-590f38f7.ckpt",
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/raft-things-802bbcfd.ckpt",
        "sintel": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/raft-sintel-fb44381e.ckpt",
        "kitti": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/raft-kitti-3a831a4b.ckpt",
    }
    _variant = _lib.VARIANT_RAFT  # pfb_raft_cfg.variant
    _engine_cls = RaftEngine  # packs the update block and runs its loop (SKFlow brings its own)

    def __init__(self, corr_levels: int = 4, corr_radius: int = 4, dropout: float = 0.0, gamma: float = 0.8,
                 max_flow: float = 400, iters: int = 32, alternate_corr: bool = False, **kwargs) -> None:
        super().__init__(output_stride=8, loss_fn=SequenceLoss(gamma, max_flow), **kwargs)
        self.corr_levels, self.corr_radius = corr_levels, corr_radius
        self.dropout, self.gamma, self.max_flow = dropout, gamma, max_flow
        self.iters, self.alternate_corr = iters, alternate_corr
        self.has_trained_on_ptlflow = True
        # backend knobs (not hparams): 0 auto, 1 SIMT fp32-accumulate kernels, 2 force the tensor-core (wgmma) kernels
        self.kernel_impl = 0
        self.strict_fp32 = True  # fp32 models: keep cuDNN off TF32 so the 1e-3 parity gate holds
        # images per encoder pass (0 = whole batch).  Smaller passes keep the 1/2-resolution intermediates of the
        # norm / activation kernels inside the 126 MB L2 instead of streaming them through HBM.
        import os as _os
        self.encoder_chunk = int(_os.environ.get("PFB_ENCODER_CHUNK", "0"))
        self.cudnn_benchmark = bool(int(_os.environ.get("PFB_CUDNN_BENCHMARK", "1")))
        # channels of the pre-processed frames handed to the first convolution (>= 3, extra channels zero): with 3,
        # cuDNN runs its own NHWC channel-padding kernel in front of the 7x7 convolution (ncu launch list r01 v15)
        self.frame_channels = int(_os.environ.get("PFB_FRAME_CHANNELS", "4"))
        # independent branches of a forward on a second stream (fork / join; parallel branches of the CUDA graph): fnet beside cnet,
        # and inside the refinement loop the flow branch of the motion encoder beside the lookup / correlation branch
        self.fork_encoders = bool(int(_os.environ.get("PFB_FORK_ENCODERS", "1")))
        self.fork_flow = bool(int(_os.environ.get("PFB_FORK_FLOW", "1")))
        self.encoder_lanes = int(_os.environ.get("PFB_ENCODER_LANES", "2"))  # 2: fnet | cnet; 3: fnet(frame 1) | fnet(frame 2) | cnet
        self._enc_tuned: set = set()
        self._engine: Optional[RaftEngine] = None
        # one CUDA graph per (input shape, dtype, iters, stream): PFB_CUDA_GRAPH=0 or model.use_cuda_graph = False -> eager launches
        self.use_cuda_graph = bool(int(_os.environ.get("PFB_CUDA_GRAPH", "1")))
        self._graphs: Dict[tuple, tuple] = {}
        self._graph_seen: Dict[tuple, int] = {}
        self.graph_capture_after = int(_os.environ.get("PFB_GRAPH_AFTER", "1"))  # eager calls of a (shape, ...) key before it is captured
        self._graph_sig = None
        self.graph_replays = 0
        self.graph_launches_replayed = 0  # this library's kernel launches replayed from graphs (bench.py: gpu_launches)
        self._build_networks()

    def _build_networks(self) -> None:
        self.hidden_dim = self.context_dim = 128
        self.fnet = BasicEncoder(output_dim=256, norm_fn="instance", dropout=self.dropout)
        self.cnet = BasicEncoder(output_dim=self.hidden_dim + self.context_dim, norm_fn="batch", dropout=self.dropout)
        self.update_block = BasicUpdateBlock(self.corr_levels, self.corr_radius, hidden_dim=self.hidden_dim)

    def freeze_bn(self) -> None:
        for m in self.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.eval()

    # -- engine lifecycle ------------------------------------------------------------------
    def _get_engine(self, dtype: torch.dtype, device: torch.device) -> RaftEngine:
        """The engine, rebuilt when what it packed (the parameters of _loop_parameters()) or what it was built for changed."""
        key = (dtype, device, self.kernel_impl, self.corr_levels, self.corr_radius,
               tuple((p.data_ptr(), p._version, p.dtype, str(p.device)) for p in self._loop_parameters()))
        eng = self._engine
        if eng is None or eng.signature != key:
            eng = self._engine_cls(self._engine_module(), self._variant, self.hidden_dim, self.context_dim, self.corr_levels,
                                   self.corr_radius, dtype, device, impl=self.kernel_impl, **self._extra_engine_args())
            eng.signature = key
            self._engine = eng
        return eng

    def _loop_parameters(self):
        """The parameters the refinement engine packs (its cache key, and the training guard of forward())."""
        return list(self.update_block.parameters())

    def _engine_module(self) -> nn.Module:
        return self.update_block

    def _extra_engine_args(self) -> Dict:
        return {}

    def _attention(self, inp: torch.Tensor, eng):
        return None

    def _correlation(self, fmap1: torch.Tensor, fmap2: torch.Tensor, inp: torch.Tensor, coords: torch.Tensor, eng):
        """(pyramid, layout, fmap1 or None) that the refinement loop reads: with alternate_corr fmap2's feature pyramid for the
        on-the-fly lookup, else the engine's volume after its before_loop.  ``inp``: the context features (llaflow's volume needs them)."""
        if self.alternate_corr:
            return ops.feature_pyramid(fmap2, self.corr_levels), 0, fmap1
        pyramid, layout = eng.build_volume(fmap1, fmap2, impl=self.kernel_impl)
        return eng.before_loop(pyramid, coords), layout, None  # csflow: the strip flow joins the start coordinates

    def _check_grid(self, h8: int, w8: int) -> None:
        """Raises ValueError, before anything is launched, for a 1/8-resolution grid (after padding) the model cannot run."""

    def _encode(self, frames: torch.Tensor, B: int, cnet_in: Optional[torch.Tensor] = None, with_fnet: bool = True):
        """frames: pixel-major [2B,Hp,Wp,3] (frame 1 of every pair first).  Both frames go through fnet as one
        batch (instance norm is per sample, extractor.py:173-176); cnet sees frame 1 only, or ``cnet_in`` when given.
        ``with_fnet = False`` runs cnet alone and returns None for both feature maps."""
        if cnet_in is None:
            cnet_in = frames[:B]
        def run(net, x):
            n = self.encoder_chunk
            if n <= 0 or x.shape[0] <= n:
                return net.forward_pm(x)
            return torch.cat([net.forward_pm(x[i : i + n]) for i in range(0, x.shape[0], n)], dim=0)

        # cuDNN autotuning: its heuristics pick an fp32 SIMT kernel for the strided 96->128 convolutions of layer3
        # (ncu launch list r01_launches_v7); benchmark mode selects per shape once.
        strict = frames.dtype == torch.float32 and self.strict_fp32
        with _cudnn_flags(self.cudnn_benchmark, not strict):
            cnet32 = self.__dict__.get("_cnet_fp32")
            own_cnet = cnet32 is None or frames.dtype == torch.float32
            tuned_key = (tuple(frames.shape), frames.dtype)
            tuned = tuned_key in self._enc_tuned  # first sight of a shape runs serially: cuDNN's autotuner times kernels then
            self._enc_tuned.add(tuned_key)
            half = frames.dtype != torch.float32
            lanes = self.encoder_lanes if (self.fork_encoders and half and with_fnet) else 1
            split_fnet = lanes >= 3  # instance norm is per sample, so fnet on the two frames of the pairs separately is exact
            fmap1 = fmap2 = None
            if lanes >= 2 and tuned and own_cnet:
                # fnet (one or two lanes) and cnet are independent, and each alternates tensor-bound convolutions with HBM-bound
                # normalise / statistics passes: on separate streams (fork / join; parallel branches of the CUDA graph) one
                # lane's convolutions fill the SMs another's memory passes leave idle
                from ... import _lib

                cur = torch.cuda.current_stream(frames.device)
                aux = _lib.thread_stream(frames.device, "aux")
                aux.wait_stream(cur)
                with torch.cuda.stream(aux):
                    cnet = run(self.cnet, cnet_in)
                if split_fnet:
                    aux2 = _lib.thread_stream(frames.device, "aux2")
                    aux2.wait_stream(cur)
                    with torch.cuda.stream(aux2):
                        fmap1 = run(self.fnet, frames[:B])
                    fmap2 = run(self.fnet, frames[B:])
                    cur.wait_stream(aux2)
                else:
                    fmaps = run(self.fnet, frames)
                cur.wait_stream(aux)
            else:
                if split_fnet:
                    fmap1, fmap2 = run(self.fnet, frames[:B]), run(self.fnet, frames[B:])
                elif with_fnet:
                    fmaps = run(self.fnet, frames)
                if own_cnet:
                    cnet = run(self.cnet, cnet_in)
            if fmap1 is None and with_fnet:
                fmap1, fmap2 = fmaps[:B], fmaps[B:]
        if cnet32 is not None and frames.dtype != torch.float32:
            # accuracy mode (enable_fp32_context): the context encoder in true fp32, its output rounded once to the storage type
            with _cudnn_flags(self.cudnn_benchmark, False):
                cnet = run(cnet32, cnet_in.float()).to(frames.dtype)
        return fmap1, fmap2, cnet

    def enable_fp32_context(self, on: bool = True) -> "RAFT":
        """Accuracy mode for f16 / bf16 models: evaluate the context encoder in true fp32 (weights as they are NOW, so call
        this before ``.half()``), everything else unchanged.  tools/f16_error_budget.py shows why this is the one stage that
        matters: its output (``net0`` / ``inp``) enters every refinement iteration, so its f16 operand rounding is a static
        perturbation that never averages out (> 90 % of the half-precision flow error); with it in fp32 the f16 pipeline
        is within north_star's 1e-2 px of the fp32 reference.  Costs a cuDNN fp32 pass over 1/3 of the encoder work, which
        is why it is not the default (bench.py reports both)."""
        import copy

        if on:
            c = copy.deepcopy(self.cnet).float().eval()
            for p_ in c.parameters():
                p_.requires_grad_(False)
            self.__dict__["_cnet_fp32"] = c  # not a registered submodule: .half() / state_dict() / parameters() do not see it
        else:
            self.__dict__.pop("_cnet_fp32", None)
        self._graphs.clear()
        return self

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        c = self.__dict__.get("_cnet_fp32")
        if c is not None:  # follow device moves, keep fp32
            dev = next(self.parameters()).device
            c.to(device=dev)
            self._graphs.clear()
        return out

    def _forward_device(self, images: torch.Tensor, flow_init: Optional[torch.Tensor], scratch: Optional[dict] = None):
        """``scratch``: a dict that owns every scratch buffer of this forward (refinement workspace, normalisation sums).  A CUDA
        graph passes its own, so that graphs replayed side by side on different streams share nothing but read-only weights."""
        if scratch is None:
            return self._forward_device_impl(images, flow_init, None)
        with ops.scratch_scope(scratch):
            return self._forward_device_impl(images, flow_init, scratch)

    def _forward_device_impl(self, images: torch.Tensor, flow_init: Optional[torch.Tensor], scratch: Optional[dict]):
        """images [B,2,3,H,W] on the device (only read) -> (flow_up fp32 [B,2,H,W], flow_small fp32 [B,2,H/8,W/8]).
        Everything in here is enqueued on the current stream with no host synchronisation and no data-dependent
        control flow, so the whole forward can be captured into one CUDA graph (``_forward_graphed``)."""
        from ...utils.utils import InputPadder

        # fused equivalent of preprocess_images(bgr_add=-0.5, bgr_mult=2, bgr_to_rgb=True, pad "replicate" two-sided)
        # (raft.py:127-135): one kernel, output already pixel-major; the caller's tensor is only read
        resizer = InputPadder(images.shape, stride=self.output_stride, pad_mode="replicate", two_side_pad=True)
        B = images.shape[0]
        frames = ops.preprocess_frames(images, resizer.tgt_size, resizer.pad_top_left, out_channels=self.frame_channels)
        fmap1, fmap2, cnet = self._encode(frames, B)
        _, H8, W8, _ = fmap1.shape
        eng = self._get_engine(fmap1.dtype, fmap1.device)
        net, inp = ops.context_split(cnet, self.hidden_dim, self.context_dim)
        coords = ops.init_coords(B, H8, W8, fmap1.device, flow_init)

        pyramid, layout, f1 = self._correlation(fmap1, fmap2, inp, coords, eng)

        orig_h, orig_w = images.shape[-2:]
        pad_top, pad_left = resizer.pad_top_left
        attention = self._attention(inp, eng)  # gma only (gma.py:181)
        flow_up, flow_small = eng.refine(pyramid, layout, net, inp, coords, self.iters, (orig_h, orig_w), (pad_top, pad_left), fmap1=f1,
                                         attention=attention, scratch=scratch, fork_flow=self.fork_flow)
        return self.postprocess_predictions(flow_up, resizer, is_flow=True), flow_small  # un-pad is a no-op: written un-padded

    # -- CUDA graph of the whole forward (SURVEY.md section 7 step 9, appendix B.9) ------------------------------
    def _graph_key(self, images: torch.Tensor, flow_init) -> tuple:
        sid = torch.cuda.current_stream(images.device).cuda_stream  # one graph (and one set of static buffers) per stream
        return (tuple(images.shape), images.dtype, str(images.device), sid, self.iters, bool(self.alternate_corr), flow_init is not None,
                self.kernel_impl, self.corr_levels, self.corr_radius, self.encoder_chunk, self.frame_channels, self.fork_encoders, self.fork_flow, self.encoder_lanes)

    def _weights_signature(self) -> tuple:
        return tuple((p.data_ptr(), p._version) for p in self.parameters()) + tuple((b.data_ptr(), b._version) for b in self.buffers())

    def _capture(self, key, images: torch.Tensor, flow_init: Optional[torch.Tensor]):
        """Two eager warm-ups, then the capture, on this library's private stream; called with the capture gate held."""
        dev = images.device
        cur = torch.cuda.current_stream(dev)
        static_in = torch.empty_like(images)
        static_init = torch.empty_like(flow_init) if flow_init is not None else None
        static_in.copy_(images)
        if static_init is not None:
            static_init.copy_(flow_init)
        from ... import _lib

        lib = _lib.load()
        scratch: dict = {}  # workspaces of this graph: owned by the cache entry, so they live exactly as long as the graph
        # the capture stream is this library's own (not from torch's pool of 32, where it could be the very stream another
        # host thread is launching on); captures are serialised, so one per device is enough
        side = _lib.private_stream(dev)
        with torch.cuda.stream(side):
            side.wait_stream(cur)
            for _ in range(2):  # eager warm-up on the capture stream: cuDNN autotune, weight packing, scratch caches
                self._forward_device(static_in, static_init, scratch)
            side.synchronize()
            n0 = lib.pfb_launch_count(-1)
            graph = torch.cuda.CUDAGraph()
            # thread_local: other host threads (pipeline slots, data loaders) keep making CUDA calls while this one captures
            with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
                flow_up, flow_small = self._forward_device(static_in, static_init, scratch)
            launches = int(lib.pfb_launch_count(-1) - n0)
        cur.wait_stream(side)
        if len(self._graphs) >= 8:  # shapes / streams come and go (infer.py, validate.py: dataset-dependent sizes)
            self._graphs.pop(next(iter(self._graphs)))
        ent = (graph, static_in, static_init, flow_up, flow_small, launches, scratch)
        self._graphs[key] = ent
        return ent

    def _forward_graphed(self, images: torch.Tensor, flow_init: Optional[torch.Tensor]):
        """One ``cudaGraphLaunch`` per forward.  The ~250 kernels of a forward (encoders, volume, 12 x 13 refinement
        launches, upsample) cost ~6 ms of host time when launched one by one; captured once per
        (shape, dtype, iters, stream) they replay from static buffers.  The parameters' storage/version is part of the
        key, so ``load_state_dict`` / ``.half()`` after a capture re-captures."""
        sig = self._weights_signature()
        if self._graph_sig != sig:
            self._graphs.clear()
            self._graph_seen.clear()
            self._graph_sig = sig
        key = self._graph_key(images, flow_init)
        ent = self._graphs.get(key)
        if ent is None and self.graph_capture_after > 0:
            # a capture costs about four forwards (two warm-ups, the capture, its first replay) and pins the forward's memory:
            # only shapes that come back are captured (infer.py / validate.py feed dataset-dependent sizes, often once each)
            seen = self._graph_seen.get(key, 0)
            if seen < self.graph_capture_after:
                if len(self._graph_seen) > 64:
                    self._graph_seen.clear()
                self._graph_seen[key] = seen + 1
                with _gate.forward():
                    return self._forward_device(images, flow_init), False
        if ent is None:
            with _gate.capture():
                ent = self._graphs.get(key) or self._capture(key, images, flow_init)  # (another thread may have got there first)
        graph, static_in, static_init, flow_up, flow_small, launches = ent[:6]
        with _gate.forward():
            static_in.copy_(images, non_blocking=True)
            if static_init is not None:
                static_init.copy_(flow_init, non_blocking=True)
            graph.replay()
        self.graph_replays += 1
        self.graph_launches_replayed += launches
        return (flow_up, flow_small), True

    def forward(self, inputs: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """Estimate optical flow between a pair of frames (eval semantics of raft.py:125-194)."""
        images = inputs["images"]
        if not images.is_cuda:
            raise RuntimeError("ptlflow_b200 runs on CUDA (sm_90a) only: move the model and inputs to the GPU. There is no CPU path.")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self._loop_parameters()) and self.training:
            raise NotImplementedError("ptlflow_b200 implements the inference hot path; call under torch.no_grad() / model.eval()")
        stride = self.output_stride
        self._check_grid(-(-images.shape[-2] // stride), -(-images.shape[-1] // stride))
        with torch.no_grad(), torch.cuda.device(images.device):
            images = images.contiguous()
            flow_init = None
            prev = inputs.get("prev_preds")
            if prev is not None and prev.get("flow_small") is not None:
                from ...utils.warm_start import forward_interpolate_batch

                flow_init = forward_interpolate_batch(prev["flow_small"]).to(device=images.device, dtype=torch.float32).contiguous()
            use_graph = self.use_cuda_graph and not torch.cuda.is_current_stream_capturing()
            if use_graph:
                (flow_up, flow_small), use_graph = self._forward_graphed(images, flow_init)  # (False: ran eagerly, fresh tensors)
            else:
                with _gate.forward():
                    flow_up, flow_small = self._forward_device(images, flow_init)
            out_dtype = inputs["images"].dtype
            # .to() / clone() give the caller fresh tensors: the graph's static outputs are overwritten by the next replay
            with _gate.forward():
                flows = flow_up.to(out_dtype) if out_dtype != torch.float32 else (flow_up.clone() if use_graph else flow_up)
                small = flow_small.to(out_dtype) if out_dtype != torch.float32 else (flow_small.clone() if use_graph else flow_small)
                fp32 = flow_up.clone() if use_graph else flow_up
            return {"flows": flows[:, None], "flow_small": small, "flows_fp32": fp32[:, None]}


class RAFTSmall(RAFT):
    pretrained_checkpoints = {
        "things": "https://github.com/hmorimitsu/ptlflow/releases/download/weights1/raft_small-things-b7d9f997.ckpt"
    }
    _variant = _lib.VARIANT_RAFT_SMALL

    def __init__(self, corr_levels: int = 4, corr_radius: int = 3, dropout: float = 0.0, gamma: float = 0.8,
                 max_flow: float = 400, iters: int = 32, alternate_corr: bool = False, **kwargs) -> None:
        super().__init__(corr_levels=corr_levels, corr_radius=corr_radius, dropout=dropout, gamma=gamma, max_flow=max_flow,
                         iters=iters, alternate_corr=alternate_corr, **kwargs)

    def _build_networks(self) -> None:
        self.hidden_dim, self.context_dim = 96, 64
        self.fnet = SmallEncoder(output_dim=128, norm_fn="instance", dropout=self.dropout)
        self.cnet = SmallEncoder(output_dim=self.hidden_dim + self.context_dim, norm_fn="none", dropout=self.dropout)
        self.update_block = SmallUpdateBlock(self.corr_levels, self.corr_radius, hidden_dim=self.hidden_dim)


@register_model
@trainable
@ptlflow_trained
class raft(RAFT):
    pass


@register_model
@trainable
@ptlflow_trained
class raft_small(RAFTSmall):
    pass
