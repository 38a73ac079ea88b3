"""FramePipeline: several frame-pair batches in flight on one GPU.

One forward of a RAFT-family model is a chain of ~250 dependent kernels that alternate between tensor-bound
(update-block convolutions), HBM-bound (encoder normalisation passes, lookup, volume) and latency-bound phases.
Two independent batches on two CUDA streams fill each other's gaps (``bench.py --inflight 2`` measures what that brings).

Each slot owns a CUDA stream, a host thread (kernel launches of one forward take ~6 ms of host time; cuDNN's
autotune cache in torch is thread-local, so the thread is long-lived and warms up once) and, through the
stream-keyed scratch caches of ``ptlflow_b200.engine`` / ``ptlflow_b200.ops``, its own workspaces.  Weights and
packed filters are shared read-only.  Results are bit-identical to sequential calls
(``tests/test_gpu_e2e.py::test_pipeline_matches_sequential``).

This is host plumbing around ``model(inputs)``; it has no counterpart in the reference, whose ``infer.py`` /
``validate.py`` loops call the model one batch at a time.
"""
from __future__ import annotations

import os
import queue
import threading
from concurrent.futures import Future
from typing import Dict, List, Optional

import torch


def _cuda_tensors(*objs):
    """Every CUDA tensor inside (possibly nested) dicts / lists / tuples."""
    for o in objs:
        if isinstance(o, torch.Tensor):
            if o.is_cuda:
                yield o
        elif isinstance(o, dict):
            yield from _cuda_tensors(*o.values())
        elif isinstance(o, (list, tuple)):
            yield from _cuda_tensors(*o)


class _Result:
    """Outputs of one submitted batch; ``get()`` waits for the slot's stream to reach the end of that batch."""

    def __init__(self, future: Future, device: torch.device):
        self._future = future
        self._device = device

    def get(self) -> Dict[str, torch.Tensor]:
        out, event = self._future.result()
        self._future = _Done((out, event))  # the Future object (also referenced by the worker's frame) lets go of the tensors
        event.synchronize()
        cur = torch.cuda.current_stream(self._device)
        for v in out.values():  # allocated on the slot's stream, consumed on the caller's
            if isinstance(v, torch.Tensor) and v.is_cuda:
                v.record_stream(cur)
        return out

    def enqueued(self) -> None:
        """Returns when the host side has finished launching the batch (the GPU may still be running it)."""
        self._future.result()


class _Done:
    def __init__(self, value):
        self._value = value

    def result(self):
        return self._value


class FramePipeline:
    def __init__(self, model: torch.nn.Module, depth: int = 2, device: Optional[torch.device] = None, prioritise_first: Optional[bool] = None):
        if depth < 1:
            raise ValueError("FramePipeline: depth must be >= 1")
        self.model = model
        self.device = device if device is not None else next(model.parameters()).device
        if self.device.type != "cuda":
            raise RuntimeError("FramePipeline needs a model on a CUDA device")
        self.depth = depth
        # prioritise_first: slot 0 on a high-priority stream.  When both slots have a kernel ready the scheduler then
        # prefers slot 0, which pulls the slots out of lockstep (identical phases compete for the same resource; a
        # tensor-bound phase next to an HBM-bound one do not).
        if prioritise_first is None:
            prioritise_first = bool(int(os.environ.get("PFB_PIPE_PRIORITY", "0")))
        self.streams = [torch.cuda.Stream(device=self.device, priority=-1 if (prioritise_first and i == 0) else 0) for i in range(depth)]
        self._queues: List[queue.Queue] = [queue.Queue() for _ in range(depth)]
        self._dev_in: List[Optional[torch.Tensor]] = [None] * depth
        self._next = 0
        self._pending: List[threading.Event] = []
        self._threads = [threading.Thread(target=self._run, args=(i,), daemon=True, name=f"pfb-slot{i}") for i in range(depth)]
        for t in self._threads:
            t.start()

    # -- worker ------------------------------------------------------------------------------
    def _run(self, slot: int) -> None:
        torch.cuda.set_device(self.device)
        stream = self.streams[slot]
        q = self._queues[slot]
        with torch.no_grad(), torch.cuda.stream(stream):
            while True:
                job = q.get()
                if job is None:
                    return
                images, extra, host_out, ready, fut, launched = job
                try:
                    stream.wait_event(ready)  # everything the caller had enqueued before submit()
                    # device-resident inputs were allocated on the caller's stream but are read on this one: tell the
                    # caching allocator, or the block could be handed back (and overwritten) while the forward still reads it
                    for t in _cuda_tensors(images, extra):
                        t.record_stream(stream)
                    if not images.is_cuda:  # pinned host frames: H2D on this slot's stream, overlapping the other slot's compute
                        buf = self._dev_in[slot]
                        if buf is None or buf.shape != images.shape or buf.dtype != images.dtype:
                            buf = torch.empty(images.shape, dtype=images.dtype, device=self.device)
                            self._dev_in[slot] = buf
                        buf.copy_(images, non_blocking=True)
                        images = buf
                    inputs = dict(extra)
                    inputs["images"] = images
                    out = self.model(inputs)
                    if host_out is not None:
                        host_out.copy_(out["flows"], non_blocking=True)
                    done = torch.cuda.Event()
                    done.record(stream)
                    fut.set_result((out, done))
                    del out
                except BaseException as e:  # noqa: BLE001 -- delivered to the caller through the future
                    fut.set_exception(e)
                finally:
                    launched.set()

    # -- caller side ---------------------------------------------------------------------------
    def submit(self, inputs: Dict[str, torch.Tensor], host_out: Optional[torch.Tensor] = None) -> _Result:
        """Enqueue ``model(inputs)`` on the next slot.  ``inputs["images"]`` may live on the device or in (pinned) host
        memory; with ``host_out`` (pinned, shape of ``flows``) the predicted flow is copied back on the slot's stream."""
        slot = self._next
        self._next = (self._next + 1) % self.depth
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(self.device))
        fut: Future = Future()
        launched = threading.Event()
        extra = {k: v for k, v in inputs.items() if k != "images"}
        self._queues[slot].put((inputs["images"], extra, host_out, ready, fut, launched))
        # only the "host side has launched it" markers are kept here: the outputs live exactly as long as the caller
        # keeps the returned _Result (a long clip must not accumulate every batch's flow on the GPU)
        self._pending = [e for e in self._pending if not e.is_set()]
        self._pending.append(launched)
        return _Result(fut, self.device)

    def drain(self) -> None:
        """Host: wait until every submitted batch has been launched; device: make the caller's current stream wait for
        all slots (so an event recorded after drain() brackets the submitted work)."""
        for e in self._pending:
            e.wait()
        self._pending.clear()
        cur = torch.cuda.current_stream(self.device)
        for s in self.streams:
            cur.wait_stream(s)

    def close(self) -> None:
        for q in self._queues:
            q.put(None)
        for t in self._threads:
            t.join(timeout=60)

    def __enter__(self) -> "FramePipeline":
        return self

    def __exit__(self, *exc) -> None:
        self.drain()
        self.close()


class FrameFeeder:
    """Decodes frame pairs on worker threads and yields host batches ready for ``FramePipeline.submit``.

    The reference's ``infer.py:178-231`` decodes with ``cv.imread`` on the critical path, one pair at a time; here the
    decode of the next batches overlaps the GPU work of the current ones.  Yields ``(indices, images)`` with ``images``
    a (pinned, when CUDA is present) ``[b,2,3,H,W]`` tensor in the reference's input convention (BGR, [0,1]); a batch
    never mixes frame sizes."""

    def __init__(self, pairs, batch: int = 8, dtype: torch.dtype = torch.float16, workers: int = 4, prefetch: int = 3, pin: Optional[bool] = None):
        self.pairs = list(pairs)
        self.batch, self.dtype, self.workers, self.prefetch = batch, dtype, workers, prefetch
        self.pin = torch.cuda.is_available() if pin is None else pin

    @staticmethod
    def _decode(path) -> torch.Tensor:
        import cv2

        img = cv2.imread(str(path), cv2.IMREAD_COLOR)
        if img is None:
            raise FileNotFoundError(f"could not read image {path}")
        return torch.from_numpy(img).permute(2, 0, 1)  # uint8 [3,H,W], BGR

    def _make_batch(self, idx: List[int]):
        from concurrent.futures import ThreadPoolExecutor

        with ThreadPoolExecutor(max_workers=self.workers) as ex:
            frames = list(ex.map(self._decode, [p for i in idx for p in self.pairs[i]]))
        groups: List[List[int]] = []
        for k, i in enumerate(idx):  # split where the frame size changes
            shp = tuple(frames[2 * k].shape)
            if tuple(frames[2 * k + 1].shape) != shp:
                raise ValueError(f"pair {i}: the two frames differ in size")
            if groups and tuple(frames[2 * (groups[-1][0] - idx[0])].shape) == shp:
                groups[-1].append(i)
            else:
                groups.append([i])
        out = []
        for g in groups:
            k0 = g[0] - idx[0]
            h, w = frames[2 * k0].shape[1:]
            buf = torch.empty((len(g), 2, 3, h, w), dtype=self.dtype)
            if self.pin:
                buf = buf.pin_memory()
            for j, i in enumerate(g):
                k = i - idx[0]
                buf[j, 0] = frames[2 * k].to(self.dtype) / 255.0
                buf[j, 1] = frames[2 * k + 1].to(self.dtype) / 255.0
            out.append((g, buf))
        return out

    def __iter__(self):
        chunks = [list(range(i, min(i + self.batch, len(self.pairs)))) for i in range(0, len(self.pairs), self.batch)]
        q: "queue.Queue" = queue.Queue(maxsize=max(1, self.prefetch))

        def produce():
            try:
                for c in chunks:
                    for item in self._make_batch(c):
                        q.put(item)
                q.put(None)
            except BaseException as e:  # noqa: BLE001 -- re-raised in the consumer
                q.put(e)

        t = threading.Thread(target=produce, daemon=True, name="pfb-feeder")
        t.start()
        while True:
            item = q.get()
            if item is None:
                break
            if isinstance(item, BaseException):
                raise item
            yield item
        t.join(timeout=60)
