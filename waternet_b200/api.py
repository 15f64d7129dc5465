"""Host-buffer convenience API: numpy uint8 images in, numpy uint8 images out.

This is the per-frame body of the reference's ``inference.py:169-233,261-323``
(preprocess -> model -> postprocess) as one call.  Host<->device copies use pinned
staging buffers on side streams and are pipelined against the kernels pass by
pass (SURVEY.md 8f.2 "pinned-memory double-buffered H2D/D2H"):

    copy-in stream   H2D pass k+1 | H2D pass k+2 | ...
    compute stream        kernels pass k | kernels pass k+1 | ...
    copy-out stream            (collective of pass k-1) D2H pass k-1 | ...

``submit()`` enqueues one batch and returns a ticket; ``wait()`` blocks until that
batch's result is in the caller's pinned buffer.  With two slots of device buffers a
caller that submits batch i+1 before waiting for batch i (a video loop) keeps the
copies of one batch entirely under the kernels of its neighbours.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

from . import _lib
from .engine import AUTO_TILE, Engine, is_auto
from .net import MODES


class _Slot:
    """Device-side staging of one in-flight batch."""

    def __init__(self):
        self.dev_in = None
        self.dev_out = None
        self.done = None      # event on the copy-out stream: the result is in the caller's pinned buffer
        self.graph = None     # CUDA graph of the kernel sequence (small frames)
        self.graph_key = None


class Enhancer:
    """A model's engine (packed weights) plus staging buffers and streams for repeated host-buffer calls.

    For small frames the ~15 kernel launches of one enhance call cost more host time than the GPU
    needs to run them; with ``cuda_graph=True`` (default for batches up to ``GRAPH_MAX_PIXELS``) the
    launch sequence is captured once per input shape into a CUDA graph and replayed.

    ``tile``: ``None`` runs whole images per pass (``Engine.enhance``).  An int or (h, w) runs the tiled forward
    (``Engine.enhance_tiled``: the same bits, with a workspace that does not grow with the image size -- for photos
    and frames too large for one pass) one image per pipelined pass, so that image i+1's copy-in runs under image
    i's kernels; it never captures a graph.  Tensor-core precisions only.  ``"auto"`` chooses per call shape
    (``Engine.auto_tile``): whole images where their workspace fits ``Engine.AUTO_WORKSPACE_BYTES`` (None: half the
    card's memory), else the tiled forward with ``Engine.DEFAULT_TILE``; whole images always with precision "fp32".
    """

    GRAPH_MAX_PIXELS = 1 << 20

    def __init__(self, model, device=None, precision: Optional[str] = None, cuda_graph: bool = True, depth: int = 2,
                 tile=None):
        if device is not None:
            model = model.to(device)
        self.model = model
        self.engine: Engine = model.engine()  # raises without CUDA: there is no CPU path
        self.mode = model._mode() if precision is None else MODES[precision]
        self.tile = tile if tile is None or is_auto(tile) else Engine._tile_hw(tile)
        if self.tile not in (None, AUTO_TILE) and self.mode == _lib.MODE_FP32_SIMT:
            raise ValueError("tile: the tiled forward runs in the tensor-core precisions only, not fp32")
        self.cuda_graph = cuda_graph
        self._slots: List[_Slot] = [_Slot() for _ in range(max(1, depth))]
        self._next = 0
        self._pin_in = None
        self._pin_out = None
        self._pin_many = None  # enhance_many's staging buffers (in, out), grown to the largest call
        dev = self.engine.device
        self._s_in = torch.cuda.Stream(dev)
        self._s_out = torch.cuda.Stream(dev)

    # ---- numpy convenience --------------------------------------------------------------------
    def __call__(self, rgb: np.ndarray) -> np.ndarray:
        """rgb: uint8 HWC or NHWC.  Returns the enhanced uint8 image(s), same layout."""
        arr = np.asarray(rgb)
        single = arr.ndim == 3
        if single:
            arr = arr[None]
        if arr.dtype != np.uint8 or arr.ndim != 4 or arr.shape[3] != 3:
            raise ValueError(f"expected uint8 (N)HWC RGB, got {arr.dtype} {arr.shape}")
        if self._pin_in is None or tuple(self._pin_in.shape) != tuple(arr.shape):
            self._pin_in = torch.empty(arr.shape, dtype=torch.uint8).pin_memory()
            self._pin_out = torch.empty(arr.shape, dtype=torch.uint8).pin_memory()
        self._pin_in.numpy()[...] = arr
        self.enhance_pinned(self._pin_in, self._pin_out)
        out = self._pin_out.numpy().copy()
        return out[0] if single else out

    def enhance_many(self, images) -> list:
        """A list of uint8 HWC images, each of its own size (a directory of photos), enhanced in one ragged call
        (``Engine.enhance_ragged`` with ``tile``, or ``Engine.DEFAULT_TILE`` when that is None or "auto"): one copy
        in through a pinned staging buffer of the total size, one call, one copy out.  Returns the list of enhanced
        images; each equals what ``self(image)`` returns.  Tensor-core precisions only."""
        if self.mode == _lib.MODE_FP32_SIMT:
            raise ValueError("enhance_many: ragged batches run in the tensor-core precisions only, not fp32")
        arrs = [np.asarray(a) for a in images]
        for i, a in enumerate(arrs):
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
                raise ValueError(f"image {i}: expected uint8 HWC RGB, got {a.dtype} {a.shape}")
        offs = np.cumsum([0] + [a.size for a in arrs]).tolist()
        total = offs[-1]
        if total == 0:
            return [a.copy() for a in arrs]
        if self._pin_many is None or self._pin_many[0].numel() < total:
            self._pin_many = (torch.empty(total, dtype=torch.uint8).pin_memory(),
                              torch.empty(total, dtype=torch.uint8).pin_memory())
        pin_in, pin_out = self._pin_many
        for a, o in zip(arrs, offs):
            pin_in.numpy()[o:o + a.size] = a.reshape(-1)
        eng = self.model.engine()  # re-packs if the parameters changed since the last call (no-op otherwise)
        dev = eng.device
        dev_in = torch.empty(total, dtype=torch.uint8, device=dev)
        dev_out = torch.empty(total, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):  # the copies and the call on the device's current stream
            dev_in.copy_(pin_in[:total], non_blocking=True)
            views = [(dev_in[o:o + a.size].view(a.shape), dev_out[o:o + a.size].view(a.shape))
                     for a, o in zip(arrs, offs)]
            tile = Engine.DEFAULT_TILE if self.tile in (None, AUTO_TILE) else self.tile
            eng.enhance_ragged([v for v, _ in views], tile=tile, mode=self.mode,
                               out_u8=[v for _, v in views])
            pin_out[:total].copy_(dev_out, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
        out = pin_out.numpy()
        return [out[o:o + a.size].reshape(a.shape).copy() for a, o in zip(arrs, offs)]

    # ---- kernels of one pass --------------------------------------------------------------------
    def _call_tile(self, n: int, h: int, w: int):
        """The tile of a call on n images of h x w: ``tile``, with "auto" resolved for that shape."""
        if self.tile != AUTO_TILE:
            return self.tile
        return Engine.auto_tile("enhance", (n, h, w), self.mode, device=self.engine.device)

    def _run_kernels(self, eng: Engine, slot: _Slot, a: int, b: int, whole: bool, tile=None, peer_out=()) -> None:
        """preprocess -> forward -> ten2arr of images [a, b) of the slot (graph replay when small), in windows of
        ``tile`` when it is not None."""
        src, dst = slot.dev_in[a:b], slot.dev_out[a:b]
        shape = tuple(slot.dev_in.shape)
        if tile is not None:
            eng.enhance_tiled(src, tile=tile, mode=self.mode, out_u8=dst)
            return
        if peer_out or not (self.cuda_graph and whole and shape[0] * shape[1] * shape[2] <= self.GRAPH_MAX_PIXELS):
            eng.enhance(src, mode=self.mode, out_u8=dst, peer_out=peer_out)
            return

        def key():  # everything a captured launch sequence has baked in
            ws = eng._ws.get("enhance")
            return (shape, self.mode, eng.f8_overflowed(), slot.dev_in.data_ptr(), slot.dev_out.data_ptr(),
                    eng._weights_key, None if ws is None else (ws.data_ptr(), ws.numel()))

        if slot.graph is None or slot.graph_key != key():
            eng.enhance(src, mode=self.mode, out_u8=dst)  # warm-up: workspace, func attributes
            torch.cuda.current_stream(eng.device).synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                eng.enhance(src, mode=self.mode, out_u8=dst)
            slot.graph, slot.graph_key = graph, key()
            return  # the warm-up call already produced this frame's result
        slot.graph.replay()

    # ---- pipelined host-buffer path ---------------------------------------------------------------
    def submit(self, pin_in: torch.Tensor, pin_out: torch.Tensor,
               on_pass: Optional[Callable[[torch.Tensor, int, int], None]] = None, exchange=None) -> _Slot:
        """Enqueue one batch: pinned uint8 NHWC host tensor -> pinned uint8 NHWC host tensor.

        The batch is processed in passes of ``engine.chunk_images`` images; pass k's H2D copy runs on the
        copy-in stream, its kernels on the current stream, and ``on_pass(dev_out[a:b], a, b)`` (e.g. the
        all-gather of that pass's output) followed by its D2H copy on the copy-out stream.  Returns a ticket
        for :meth:`wait`; neither ``pin_in`` nor ``pin_out`` may be touched before that.

        ``exchange``: a :class:`waternet_b200.dist.PeerGather` -- the multi-GPU all-gather of the output fused into the
        kernels: every pass's last launch stores its output into all ranks' buffers as well (``exchange.addresses``),
        ``exchange.signal()`` follows the last pass on the compute stream and ``exchange.wait()`` the last D2H copy
        on the copy-out stream.  With ``tile`` "auto" a batch that would run in windows refuses ``exchange``.
        """
        if pin_in.dtype != torch.uint8 or pin_in.dim() != 4 or pin_in.shape[3] != 3 or pin_in.shape != pin_out.shape:
            raise ValueError(f"expected uint8 (N,H,W,3) pinned tensors of one shape, got {tuple(pin_in.shape)}")
        tile = self._call_tile(*pin_in.shape[:3])
        if exchange is not None and tile is not None:
            raise ValueError("exchange: the fused multi-GPU exchange is not available with tile")
        eng = self.model.engine()  # re-packs if the parameters changed since the last call (no-op otherwise)
        dev = eng.device
        slot = self._slots[self._next % len(self._slots)]
        self._next += 1
        if slot.done is not None:
            slot.done.synchronize()  # back-pressure: the previous user of these buffers has been delivered
        shape = tuple(pin_in.shape)
        if slot.dev_in is None or tuple(slot.dev_in.shape) != shape:
            slot.graph = None
            slot.dev_in = torch.empty(shape, dtype=torch.uint8, device=dev)
            slot.dev_out = torch.empty(shape, dtype=torch.uint8, device=dev)
        n, h, w, _ = shape
        cur = torch.cuda.current_stream(dev)
        if n * h * w == 0:
            if exchange is not None:  # an empty local batch still takes part in the step's completion protocol
                exchange.signal()
                exchange.wait()
            slot.done = torch.cuda.Event()
            slot.done.record(cur)
            return slot
        nb = 1 if tile is not None else eng.chunk_images(n, h, w)
        self._s_in.wait_stream(cur)   # whatever the caller enqueued before (e.g. filling pin_in on the device side)
        self._s_out.wait_stream(cur)
        for a in range(0, n, nb):
            b = min(n, a + nb)
            with torch.cuda.stream(self._s_in):
                slot.dev_in[a:b].copy_(pin_in[a:b], non_blocking=True)
                ev_in = torch.cuda.Event()
                ev_in.record(self._s_in)
            cur.wait_event(ev_in)
            self._run_kernels(eng, slot, a, b, whole=(a == 0 and b == n), tile=tile,
                              peer_out=exchange.addresses(a) if exchange is not None else ())
            if exchange is not None and b == n:
                exchange.signal()
            ev_k = torch.cuda.Event()
            ev_k.record(cur)
            with torch.cuda.stream(self._s_out):
                self._s_out.wait_event(ev_k)
                if on_pass is not None:
                    on_pass(slot.dev_out[a:b], a, b)
                pin_out[a:b].copy_(slot.dev_out[a:b], non_blocking=True)
                if exchange is not None and b == n:
                    exchange.wait()
        slot.done = torch.cuda.Event()
        slot.done.record(self._s_out)
        return slot

    def wait(self, ticket: _Slot) -> None:
        if ticket.done is not None:
            ticket.done.synchronize()

    def enhance_pinned(self, pin_in: torch.Tensor, pin_out: torch.Tensor, on_pass=None, exchange=None) -> None:
        """Pinned uint8 NHWC host tensor -> pinned uint8 NHWC host tensor; returns when ``pin_out`` is complete."""
        self.wait(self.submit(pin_in, pin_out, on_pass=on_pass, exchange=exchange))
        torch.cuda.current_stream(self.engine.device).wait_stream(self._s_out)
