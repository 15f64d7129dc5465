"""Per-device engine: owns the C-ABI handle, packed weights and workspaces.

torch is plumbing here (device memory, streams); all arithmetic happens in
libwaternet_b200.so.
"""
from __future__ import annotations

import ctypes
import threading
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

_engines: Dict[int, "Engine"] = {}
_engines_lock = threading.Lock()
# scratch buffers are shared by every engine of a device (all work is stream-ordered on the caller's stream)
_ws_pool: Dict[int, Dict[str, torch.Tensor]] = {}


def _require_cuda(device=None) -> torch.device:
    if not torch.cuda.is_available():
        raise _lib.WaterNetLibraryError(
            "waternet_b200 needs a CUDA device (H100, sm_90a); none is visible and there is no CPU fallback")
    dev = torch.device("cuda" if device is None else device)
    if dev.type != "cuda":
        raise _lib.WaterNetLibraryError(f"waternet_b200 runs on CUDA devices only, got {dev}")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def get_engine(device=None) -> "Engine":
    """The device's shared engine: preprocess / postprocess and callers that pack weights themselves."""
    dev = _require_cuda(device)
    with _engines_lock:
        eng = _engines.get(dev.index)
        if eng is None:
            eng = Engine(dev)
            _engines[dev.index] = eng
        return eng


def new_engine(device=None) -> "Engine":
    """A private engine (its own C-ABI handle, i.e. its own packed-weight slot) for one model on one device.

    Every ``WaterNet`` / ``ConfidenceMapGenerator`` / ``Refiner`` instance owns one per device, so two models on
    a device never evict -- or silently run with -- each other's packed weights.
    """
    return Engine(_require_cuda(device))


TILE_HALO = 13  # receptive-field radius of WaterNet (csrc/tiling.cuh kTileHalo)


def tile_geometry(h: int, w: int, tile_h: int, tile_w: int) -> dict:
    """The window rule of wn_enhance_u8_tiled (csrc/tiling.cuh) restated for callers that plan or check a tiled
    call: balanced tile size and count per axis, window size, and each window's origin and kept rectangle."""
    def axis(size, tile):
        count = -(-size // tile)
        t = -(-size // count)
        win = min(size, t + 2 * TILE_HALO)
        spans = [(i * t, min(size, (i + 1) * t)) for i in range(count)]
        starts = [min(max(k0 - TILE_HALO, 0), size - win) for k0, _ in spans]
        return t, count, win, spans, starts
    th, ny, win_h, rows, ys = axis(h, tile_h)
    tw, nx, win_w, cols, xs = axis(w, tile_w)
    return {"th": th, "tw": tw, "ny": ny, "nx": nx, "win_h": win_h, "win_w": win_w,
            "windows": [(ys[i], xs[j], rows[i], cols[j]) for i in range(ny) for j in range(nx)]}


def covering_windows(g: dict, y: int, x: int) -> Tuple[range, range]:
    """The windows whose extent contains pixel (y, x) of an image with ``tile_geometry`` ``g``: (tile rows, tile
    columns), as ranges (csrc/tiling.cuh tile_cover, which the windowed backward folds input gradients by).  A
    window's origin does not decrease along an axis, so the windows containing a row form one run."""
    def axis(v, size, t, count, win):
        hi = count - 1 if v >= size - win else min(count - 1, (v + TILE_HALO) // t)
        first = v - win + 1  # origin >= first
        lo = 0 if first <= 0 else -(-(first + TILE_HALO) // t)
        return range(lo, hi + 1)
    h = g["windows"][-1][2][1]
    w = g["windows"][-1][3][1]
    return axis(y, h, g["th"], g["ny"], g["win_h"]), axis(x, w, g["tw"], g["nx"], g["win_w"])


DEFAULT_PASS_PIXELS = 8 << 20  # max_pass_pixels = 0
TRAIN_PASS_PIXELS = 2 << 20    # max_pass_pixels = 0 of the windowed backward (wn_backward_tiled)
RAGGED_WINDOW_BYTES = 72       # csrc/tiling.cuh RaggedWindow: one descriptor per window
RAGGED_IMAGE_BYTES = 40        # csrc/common.cuh RaggedImage: one per image


def ragged_plan(sizes, tile_h: int, tile_w: int, max_pass_pixels: int = 0) -> list:
    """The pass plan of wn_enhance_u8_ragged (csrc/tiling.cuh ragged_plan) restated for callers that plan or check
    a ragged call.  ``sizes``: [(h, w), ...].  Returns the passes in order, each a dict with ``slot`` (h, w) and
    ``windows``: dicts with the image index ``img``, origin ``ys``, ``xs``, valid extent ``vh``, ``vw`` and kept
    ``rows`` (ky0, ky1) and ``cols`` (kx0, kx1)."""
    limit = max_pass_pixels or DEFAULT_PASS_PIXELS
    wins = []
    for i, (h, w) in enumerate(sizes):
        g = tile_geometry(h, w, tile_h, tile_w)
        wins += [{"img": i, "ys": ys, "xs": xs, "vh": g["win_h"], "vw": g["win_w"], "rows": rows, "cols": cols}
                 for ys, xs, rows, cols in g["windows"]]
    wins.sort(key=lambda r: (-r["vh"], -r["vw"]))  # stable: image and window order within a shape
    passes, cur, valid = [], None, 0
    for r in wins:
        if cur is not None:
            cnt = len(cur["windows"]) + 1
            sh, sw = max(cur["slot"][0], r["vh"]), max(cur["slot"][1], r["vw"])
            v = valid + r["vh"] * r["vw"]
            if cnt <= 65535 and cnt * sh * sw <= limit and 4 * (cnt * sh * sw - v) <= cnt * sh * sw:
                cur["windows"].append(r)
                cur["slot"], valid = (sh, sw), v
                continue
            passes.append(cur)
        cur, valid = {"slot": (r["vh"], r["vw"]), "windows": [r]}, r["vh"] * r["vw"]
    if cur is not None:
        passes.append(cur)
    return passes


def ragged_train_calls(sizes, max_pass_pixels: int) -> list:
    """How ``Engine.forward_train_ragged`` groups images of ``sizes`` [(h, w), ...] into training calls:
    ``ragged_plan`` at ``max_pass_pixels`` slot pixels per pass with a tile as large as the largest image, so that
    every image is one window and every pass one call of wn_forward_train_ragged (n x slot pixels <= the limit, at
    most 65535 images, at most 25 % padding when a call holds more than one image).  Returns one list of image
    indices per call, in call order."""
    if not sizes:
        return []
    th, tw = max(h for h, _ in sizes), max(w for _, w in sizes)
    return [[r["img"] for r in p["windows"]] for p in ragged_plan(sizes, th, tw, max_pass_pixels)]


VGG_HALO = 128                  # input pixels a perceptual-loss window reads beyond its features, per side
VGG_SUPPORT = (-118, 133)       # input rows (columns) conv5_4 feature i depends on: [16 i - 118, 16 i + 133]
VGG_PASS_PIXELS = 2 << 20       # max_pass_pixels = 0 of wn_perceptual_loss
VGG_MAX_PIXELS = 8 << 20        # cap on a window and on max_pass_pixels
VGG_SEED_BLOCKS = 16            # float64 loss partials per window
# (cin, cout) of VGG19's 16 convolutions in features order (csrc/vgg.cu kVggFwd), all 3 x 3
VGG_CONVS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 256), (256, 512),
             (512, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512))
# the 20 launches of the VGG19 forward in features order: (convolution index or -1 for a max-pool, level, channels)
VGG_STEPS = ((0, 0, 64), (1, 0, 64), (-1, 1, 64), (2, 1, 128), (3, 1, 128), (-1, 2, 128), (4, 2, 256), (5, 2, 256),
             (6, 2, 256), (7, 2, 256), (-1, 3, 256), (8, 3, 512), (9, 3, 512), (10, 3, 512), (11, 3, 512),
             (-1, 4, 512), (12, 4, 512), (13, 4, 512), (14, 4, 512), (15, 4, 512))


def vgg_tile_hw(tile) -> Tuple[int, int]:
    """``tile`` of the perceptual loss as (tile_h, tile_w): None -> (0, 0), one window per image."""
    if tile is None:
        return 0, 0
    th, tw = (tile, tile) if isinstance(tile, int) else tile
    if th <= 0 or tw <= 0:
        raise ValueError(f"perceptual-loss tile must be positive, got {tile}")
    return int(th), int(tw)


def perceptual_windows(size: int, tile: int) -> list:
    """The window rule of wn_perceptual_loss (csrc/vgg.cu) along one axis of ``size`` pixels: a list of (start, end,
    f0, f1), the input pixels [start, end) a window reads and the features [f0, f1) it owns.  ``tile`` 0: one window."""
    f = size // 16
    q = min(f, -(-tile // 16)) if tile > 0 else f
    count = -(-f // q)
    return [(max(0, 16 * k * q - VGG_HALO), min(size, 16 * (k + 1) * q + VGG_HALO), k * q, min(f, (k + 1) * q))
            for k in range(count)]


def perceptual_passes(n: int, h: int, w: int, tile_h: int, tile_w: int, max_pass_pixels: int = 0) -> list:
    """The passes of wn_perceptual_loss: classes of windows of one extent (runs of equal extent per axis), each split
    into passes of at most ``max_pass_pixels`` window pixels.  Returns [(count, win_h, win_w), ...] in order."""
    def runs(wins):
        out = []
        for s, e, _, _ in wins:
            if out and out[-1][1] == e - s:
                out[-1][0] += 1
            else:
                out.append([1, e - s])
        return out
    limit = max_pass_pixels or VGG_PASS_PIXELS
    passes = []
    for ny, wh in runs(perceptual_windows(h, tile_h)):
        for nx, ww in runs(perceptual_windows(w, tile_w)):
            total = n * ny * nx
            per = min(65535, max(1, limit // (wh * ww)))
            passes += [(min(per, total - w0), wh, ww) for w0 in range(0, total, per)]
    return passes


def perceptual_loss_workspace_bytes(n: int, h: int, w: int, tile_h: int, tile_w: int, max_pass_pixels: int = 0) -> int:
    """wn_perceptual_loss_workspace_bytes restated: 0 for rejected arguments, else the float64 partials of every
    window plus the largest pass (act0, two scratch buffers, ref's conv5_4 and the 20 saved launch outputs, each 1 KiB
    aligned) plus 1 KiB."""
    if (n <= 0 or n > 65535 or h < 16 or w < 16 or tile_h < 0 or tile_w < 0 or (tile_h == 0) != (tile_w == 0)
            or max_pass_pixels < 0 or max_pass_pixels > VGG_MAX_PIXELS or h * w > 0x7fffffff // 3):
        return 0
    a1k = lambda v: -(-v // 1024) * 1024
    passes = perceptual_passes(n, h, w, tile_h, tile_w, max_pass_pixels)
    if any(wh * ww > VGG_MAX_PIXELS for _, wh, ww in passes):
        return 0
    windows = sum(c for c, _, _ in passes)

    def pass_bytes(c, wh, ww):
        steps = [(wh >> lv) * (ww >> lv) * ch * 4 for _, lv, ch in VGG_STEPS]
        scratch = max([wh * ww * 64] + steps)
        return sum(a1k(c * b) for b in [wh * ww * 64, scratch, scratch, steps[-1]] + steps)
    return a1k(windows * VGG_SEED_BLOCKS * 8) + max(pass_bytes(*p) for p in passes) + 1024


AUTO_TILE = "auto"  # the value of tile / grad_tile that leaves the choice to Engine.auto_tile, call by call


def is_auto(tile, name: str = "tile") -> bool:
    """Whether the setting ``tile`` (named ``name`` in errors) is "auto"; any other string raises ValueError."""
    if isinstance(tile, str):
        if tile != AUTO_TILE:
            raise ValueError(f"{name} must be None, {AUTO_TILE!r}, an int or (h, w); got {tile!r}")
        return True
    return False


def _stream_ptr(device: torch.device) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


# ---- the ctypes arrays the C ABI takes
def _strides(tensors) -> ctypes.Array:
    """The element strides of ``tensors``, flattened ({sN, sC, sH, sW} each): in_strides of the C ABI."""
    return (ctypes.c_int64 * (4 * len(tensors)))(*[s for t in tensors for s in t.stride()])


def _sizes(sizes) -> Tuple[ctypes.Array, ctypes.Array]:
    """[(h, w), ...] -> the height and width arrays of the ragged calls (one entry at least)."""
    n = max(1, len(sizes))
    return (ctypes.c_int * n)(*[int(h) for h, _ in sizes]), (ctypes.c_int * n)(*[int(w) for _, w in sizes])


def _ptrs(tensors) -> ctypes.Array:
    """The device addresses of ``tensors`` (NULL for None) as an array of pointers."""
    return (ctypes.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])


def _grads_array(grads, first: int = 0) -> ctypes.Array:
    """The NUM_PARAMS parameter-gradient pointers with ``grads`` (tensors or None) at entries first, first + 1, ...
    and NULL elsewhere: the entries of a sub-module start at its first state-dict entry."""
    arr = (ctypes.c_void_p * _lib.NUM_PARAMS)()
    arr[first:first + len(grads)] = [None if t is None else t.data_ptr() for t in grads]
    return arr


def _require_workspace(nbytes: int, message: str) -> int:
    """``nbytes`` from a workspace function, which returns 0 for the arguments its call rejects: then raise."""
    if nbytes == 0:
        raise _lib.WaterNetLibraryError(message)
    return nbytes


class Engine:
    def __init__(self, device: torch.device):
        self.lib = _lib.load()
        self.device = device
        handle = ctypes.c_void_p()
        _lib.check(self.lib.wn_create(device.index, ctypes.byref(handle)), "wn_create")
        self.handle = handle
        self._ws = _ws_pool.setdefault(device.index, {})
        self._weights_key = None
        self._weights_keepalive = None

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.wn_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # ---- plumbing ----------------------------------------------------------
    def _call(self, name: str, *args, stream: bool = True) -> None:
        """``self.lib.<name>(handle, *args, current stream)`` on the engine's device (no stream argument without
        ``stream``); raises WaterNetLibraryError when it returns an error code."""
        with torch.cuda.device(self.device):
            if stream:
                args += (_stream_ptr(self.device),)
            rc = getattr(self.lib, name)(self.handle, *args)
        _lib.check(rc, name)

    def _workspace(self, tag: str, nbytes: int) -> torch.Tensor:
        buf = self._ws.get(tag)
        if buf is None or buf.numel() < nbytes:
            self._ws[tag] = None
            buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=self.device)
            self._ws[tag] = buf
        return buf

    def release_workspaces(self) -> None:
        self._ws.clear()

    def chunk_images(self, n: int, h: int, w: int) -> int:
        """Images per pass of the tensor-core forward for a batch of ``n`` (wn_forward_chunk_images)."""
        return max(1, int(self.lib.wn_forward_chunk_images(self.handle, n, h, w)))

    def set_chunk_pixels(self, max_pixels: int) -> None:
        """Lower the per-pass pixel cap (0 = default 8 Mi); tests force the multi-pass path with it."""
        self._call("wn_set_chunk_pixels", int(max_pixels), stream=False)

    def set_train_mode(self, mode: int) -> None:
        """The arithmetic of this handle's training calls (wn_set_train_mode): MODE_BF16X3 or MODE_BF16.  Every
        training method below sets it from its ``train_mode`` argument first, so a backward runs under the mode its
        caller passes (the mode of the matching forward), whatever another module did on this handle in between."""
        self._call("wn_set_train_mode", int(mode), stream=False)

    def f8_overflowed(self) -> bool:
        """True once the fp8-correction mode saw an activation beyond the e4m3 range.  The batch that did was
        recomputed by the bf16x3 kernels within the same call; from then on the handle uses those kernels
        directly until new weights are packed (wn_f8_overflowed).  Valid after the stream has been synchronised."""
        return bool(self.lib.wn_f8_overflowed(self.handle))

    @property
    def launch_count(self) -> int:
        return int(self.lib.wn_launch_count(self.handle))

    def enable_timing(self, on: bool = True) -> None:
        self._call("wn_enable_timing", 1 if on else 0, stream=False)

    def read_timings(self):
        """(ms[slot], count[slot]) accumulated since the last read; synchronises the device first."""
        torch.cuda.synchronize(self.device)
        ms = (ctypes.c_float * _lib.NUM_TIMING_SLOTS)()
        cnt = (ctypes.c_int * _lib.NUM_TIMING_SLOTS)()
        self._call("wn_read_timings", ms, cnt, stream=False)
        return list(ms), list(cnt)

    # ---- weights -------------------------------------------------------------
    def pack_weights(self, params: Sequence[torch.Tensor], key=None) -> None:
        """params: the 34 tensors in state-dict order (net.py:12-42,62-70,94-97)."""
        if len(params) != _lib.NUM_PARAMS:
            raise ValueError(f"expected {_lib.NUM_PARAMS} parameter tensors, got {len(params)}")
        if key is not None and key == self._weights_key:
            return
        staged = [p.detach().to(device=self.device, dtype=torch.float32).contiguous() for p in params]
        self._call("wn_pack_weights", _ptrs(staged))
        self._weights_keepalive = staged  # until the async pack kernels have consumed them
        self._weights_key = key

    # ---- forward -------------------------------------------------------------
    def forward(self, x, wb, he, gc, mode: int = _lib.MODE_DEFAULT, out: Optional[torch.Tensor] = None):
        """WaterNet.forward (net.py:99-108) on (N,3,H,W) fp32 CUDA tensors of any strides."""
        ins = self._check_inputs((x, wb, he, gc))
        n, _, h, w = ins[0].shape
        if out is None:
            out = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
        if n == 0 or h == 0 or w == 0:  # empty batch: nothing to launch (torch's convs return empty too)
            return out
        ws = self._workspace("forward", self.lib.wn_forward_workspace_bytes(n, h, w, mode))
        self._call("wn_forward", *(t.data_ptr() for t in ins), _strides(ins), out.data_ptr(), n, h, w, mode,
                   ws.data_ptr(), ws.numel())
        return out

    def _check_inputs(self, tensors):
        ins = []
        for t in tensors:
            if t.device != self.device:
                raise ValueError(f"input on {t.device}, engine on {self.device}")
            if t.dim() != 4 or t.shape[1] != 3:
                raise ValueError(f"expected (N,3,H,W) inputs, got {tuple(t.shape)}")
            ins.append(t.detach() if t.dtype == torch.float32 else t.detach().float())
        for t in ins[1:]:
            if t.shape != ins[0].shape:
                raise ValueError("the inputs must have the same shape")
        return ins

    def confidence_maps(self, x, wb, he, gc, mode: int = _lib.MODE_DEFAULT) -> torch.Tensor:
        """ConfidenceMapGenerator.forward (net.py:45-56): the three sigmoid maps as one (N,3,H,W) tensor."""
        ins = self._check_inputs((x, wb, he, gc))
        n, _, h, w = ins[0].shape
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
        if out.numel() == 0:
            return out
        ws = self._workspace("forward", self.lib.wn_submodule_workspace_bytes(n, h, w, mode))
        self._call("wn_confidence_maps", *(t.data_ptr() for t in ins), _strides(ins), out.data_ptr(), n, h, w, mode,
                   ws.data_ptr(), ws.numel())
        return out

    def refine(self, which: int, x, xbar, mode: int = _lib.MODE_DEFAULT) -> torch.Tensor:
        """Refiner.forward (net.py:75-80) of refiner ``which`` (0 wb, 1 ce, 2 gc) of the packed state dict."""
        ins = self._check_inputs((x, xbar))
        n, _, h, w = ins[0].shape
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
        if out.numel() == 0:
            return out
        ws = self._workspace("forward", self.lib.wn_submodule_workspace_bytes(n, h, w, mode))
        self._call("wn_refine", int(which), *(t.data_ptr() for t in ins), _strides(ins), out.data_ptr(), n, h, w,
                   mode, ws.data_ptr(), ws.numel())
        return out

    LAYER_CHANNELS = (128, 128, 128, 64, 64, 64, 64, 3, 96, 96, 9)

    def debug_layer(self, x, wb, he, gc, layer: int, mode: int) -> torch.Tensor:
        """Test aid (wn_debug_forward_layer): an intermediate activation as fp32 (N,C,H,W)."""
        ins = [t.detach().float() for t in (x, wb, he, gc)]
        n, _, h, w = ins[0].shape
        dst = torch.empty((n, self.LAYER_CHANNELS[layer], h, w), dtype=torch.float32, device=self.device)
        ws = self._workspace("forward", self.lib.wn_forward_workspace_bytes(n, h, w, mode))
        self._call("wn_debug_forward_layer", *(t.data_ptr() for t in ins), _strides(ins), n, h, w, mode, layer,
                   dst.data_ptr(), ws.data_ptr(), ws.numel())
        return dst

    # ---- training step (wn_forward_train / wn_backward) ---------------------------------------
    TRAIN_MAX_PIXELS = 8 << 20
    TRAIN_MAX_IMAGES = 65535

    def _param_grads(self, shapes, written: bool):
        """fp32 tensors of ``shapes`` for parameter gradients: uninitialised when a library call writes them, else
        zeros (nothing to run has zero gradients)."""
        make = torch.empty if written else torch.zeros
        return [make(tuple(s), dtype=torch.float32, device=self.device) for s in shapes]

    def _sum_in_order(self, shapes, calls, run):
        """The parameter gradients of ``shapes`` summed over ``calls`` in order: ``run(call, dst)`` makes one library
        call that writes its gradients into ``dst``; the first call writes the result, each later one a scratch set
        that is added to it in call order (deterministic)."""
        grads = self._param_grads(shapes, bool(calls))
        part = grads if len(calls) <= 1 else [torch.empty_like(t) for t in grads]
        for k, call in enumerate(calls):
            run(call, grads if k == 0 else part)
            if k > 0:
                torch._foreach_add_(grads, part)
        return grads

    @classmethod
    def _train_slice_bounds(cls, n: int, h: int, w: int) -> list:
        """The slices [(a, b), ...] of ``_train_slices`` for n images of h x w (at most TRAIN_MAX_PIXELS)."""
        per = min(cls.TRAIN_MAX_IMAGES, max(1, cls.TRAIN_MAX_PIXELS // (h * w)))
        return [(a, min(n, a + per)) for a in range(0, n, per)]

    def _train_slices(self, what: str, lead, ins, workspace_bytes, too_large: str, train_mode: int):
        """``ins`` in slices of at most TRAIN_MAX_PIXELS and TRAIN_MAX_IMAGES, each one call of ``what`` (``lead``
        before the inputs) with a workspace of its own of ``workspace_bytes(n, h, w)`` bytes.  Returns (out, [(a, b,
        workspace), ...]), or (out, None) for an empty batch.  One image over TRAIN_MAX_PIXELS raises ``too_large``
        with ``{h}`` and ``{w}`` filled in."""
        self.set_train_mode(train_mode)
        n, _, h, w = ins[0].shape
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
        if out.numel() == 0:
            return out, None
        if h * w > self.TRAIN_MAX_PIXELS:
            raise _lib.WaterNetLibraryError(too_large.format(h=h, w=w))
        saved = []
        for a, b in self._train_slice_bounds(n, h, w):
            part = [t[a:b] for t in ins]
            ws = torch.empty(workspace_bytes(b - a, h, w), dtype=torch.uint8, device=self.device)
            self._call(what, *lead, *(t.data_ptr() for t in part), _strides(part), out[a:b].data_ptr(), b - a, h, w,
                       ws.data_ptr(), ws.numel())
            saved.append((a, b, ws))
        return out, saved

    def _slices_backward(self, what: str, lead, first: int, grad, saved, shapes, want_inputs, train_mode: int):
        """The backward of the slices of ``_train_slices``: one call of ``what`` per slice (``lead`` before the
        gradient), the parameter gradients of ``shapes`` (state-dict entries first, first + 1, ...) summed in slice
        order, and the input gradients asked for by ``want_inputs`` (None where not)."""
        self.set_train_mode(train_mode)
        g = grad.detach().to(self.device, torch.float32).contiguous()
        n, _, h, w = g.shape
        gin = [torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device) if want else None
               for want in want_inputs]

        def run(call, dst):
            a, b, ws = call
            gin_arr = _ptrs([None if t is None else t[a:b] for t in gin]) if any(want_inputs) else None
            self._call(what, *lead, g[a:b].data_ptr(), _grads_array(dst, first), gin_arr, b - a, h, w, ws.data_ptr(),
                       ws.numel())
        return self._sum_in_order(shapes, saved or [], run), gin

    def forward_train(self, x, wb, he, gc, train_mode: int = _lib.MODE_BF16X3):
        """Tensor-core forward that keeps every activation.  Returns (out, saved workspaces).

        wn_forward_train takes at most TRAIN_MAX_PIXELS and TRAIN_MAX_IMAGES per call; a larger batch runs as several
        calls over slices of the batch, each with its own workspace (~5.6 KB per pixel in total, like the reference's autograd graph)."""
        ins = self._check_inputs((x, wb, he, gc))
        return self._train_slices(
            "wn_forward_train", (), ins, self.lib.wn_train_workspace_bytes,
            "a forward pass that keeps its activations for autograd holds ~5.6 KB per pixel: one {h}x{w} image exceeds "
            f"the {self.TRAIN_MAX_PIXELS >> 20} Mi-pixel limit of wn_forward_train.  For inference wrap the call in "
            "torch.no_grad()", train_mode)

    def backward(self, grad_out: torch.Tensor, saved, shapes, want_input_grads: bool = False, train_mode: int = _lib.MODE_BF16X3):
        """d(loss)/d(out) + the workspaces of forward_train -> the 34 parameter gradients (state-dict order)
        and, on request, the gradients of the four input images.  Batch slices are processed in order and their
        parameter gradients added in that order (deterministic).  ``train_mode``: that of the forward."""
        grads, gin = self._slices_backward("wn_backward", (), 0, grad_out, saved, shapes, (want_input_grads,) * 4,
                                           train_mode)
        return (grads, gin) if want_input_grads else grads

    # wn_debug_backward_layer's buffers 0..24 (include/waternet_b200.h): act0, a1..a7, cm, r1, r2, refined, g8, gr3 and
    # the outputs of the 11 data-gradient launches cmg.conv8 .. cmg.conv2, refiners conv3, conv2, cmg.conv1, refiners conv1
    BACKWARD_BUFFER_CHANNELS = (16, 128, 128, 128, 64, 64, 64, 64, 3, 96, 96, 9, 16, 16,
                                64, 64, 64, 64, 128, 128, 128, 96, 96, 32, 32)

    def debug_backward_layer(self, workspace: torch.Tensor, shape, buffer: int, stack: int = -1, which: int = 0,
                             grad: Optional[torch.Tensor] = None, grads=None, train_mode: int = _lib.MODE_BF16X3) -> torch.Tensor:
        """Test aid (wn_debug_backward_layer): buffer ``buffer`` of the training backward as fp32 (N,C,H,W).

        ``workspace`` is the workspace of one slice that ``forward_train`` (stack -1), ``confidence_maps_train`` (0)
        or ``refine_train(which)`` (1) has just filled, ``shape`` = (n, h, w) of that slice.  ``grad``: d(loss)/d(out)
        (d(maps) for the cmg) for the seeds and launches, buffers 12 and up.  ``grads``: 34 fp32 tensors or None
        (None where the stack writes nothing) that receive the parameter gradients of the layers before a
        data-gradient launch, buffers 14 and up.  ``train_mode``: that of the forward that filled the workspace."""
        self.set_train_mode(train_mode)
        n, h, w = shape
        dst = torch.empty((n, self.BACKWARD_BUFFER_CHANNELS[buffer], h, w), dtype=torch.float32, device=self.device)
        g = None if grad is None else grad.detach().to(self.device, torch.float32).contiguous()
        self._call("wn_debug_backward_layer", int(stack), int(which), int(buffer), None if g is None else g.data_ptr(),
                   None if grads is None else _grads_array(grads), n, h, w, dst.data_ptr(), workspace.data_ptr(),
                   workspace.numel())
        return dst

    # ---- the sub-modules under autograd (wn_confidence_maps_train / _backward, wn_refine_train / _backward) --------
    STACK_CMG, STACK_REFINER = 0, 1

    def _submodule_train_slices(self, what: str, lead, stack: int, ins, train_mode: int):
        """``_train_slices`` of one stack (wn_submodule_train_workspace_bytes of ``stack`` per slice)."""
        return self._train_slices(
            what, lead, ins, lambda n, h, w: self.lib.wn_submodule_train_workspace_bytes(n, h, w, stack),
            f"{what}: one {{h}}x{{w}} image exceeds the {self.TRAIN_MAX_PIXELS} pixels of one training call", train_mode)

    def confidence_maps_train(self, x, wb, he, gc, train_mode: int = _lib.MODE_BF16X3):
        """``confidence_maps`` in the arithmetic of training (``train_mode``), keeping the activations of the cmg stack
        (wn_confidence_maps_train).  Returns (maps, saved workspaces) for ``confidence_maps_backward``."""
        ins = self._check_inputs((x, wb, he, gc))
        return self._submodule_train_slices("wn_confidence_maps_train", (), self.STACK_CMG, ins, train_mode)

    def confidence_maps_backward(self, grad_maps, saved, shapes, want_inputs=(False,) * 4, train_mode: int = _lib.MODE_BF16X3):
        """d(loss)/d(maps) + the workspaces of ``confidence_maps_train`` -> the 16 cmg parameter gradients
        (state-dict order) and the gradients of x, wb, he, gc where ``want_inputs`` asks for them (else None)."""
        return self._slices_backward("wn_confidence_maps_backward", (), 0, grad_maps, saved, shapes, want_inputs,
                                     train_mode)

    def refine_train(self, which: int, x, xbar, train_mode: int = _lib.MODE_BF16X3):
        """``refine`` in the arithmetic of training (``train_mode``), keeping the activations of the refiner stack
        (wn_refine_train).  Returns (out, saved workspaces) for ``refine_backward``."""
        ins = self._check_inputs((x, xbar))
        return self._submodule_train_slices("wn_refine_train", (int(which),), self.STACK_REFINER, ins, train_mode)

    def refine_backward(self, which: int, grad_out, saved, shapes, want_inputs=(False, False), train_mode: int = _lib.MODE_BF16X3):
        """d(loss)/d(out) + the workspaces of ``refine_train`` -> the 6 parameter gradients of refiner ``which``
        (state-dict order) and the gradients of x, xbar where ``want_inputs`` asks for them (else None)."""
        return self._slices_backward("wn_refine_backward", (int(which),), 16 + 6 * int(which), grad_out, saved, shapes,
                                     want_inputs, train_mode)

    # ---- preprocess / postprocess ----------------------------------------------
    def preprocess(self, rgb_u8: torch.Tensor, tensors: bool = True, images: bool = False):
        """rgb_u8: uint8 (N,H,W,3) CUDA tensor.  Returns dict with the requested outputs.

        tensors -> 'x','wb','he','gc' fp32 (N,3,H,W); images -> 'wb_u8','he_u8','gc_u8' uint8 NHWC.
        """
        if rgb_u8.dtype != torch.uint8 or rgb_u8.dim() != 4 or rgb_u8.shape[3] != 3:
            raise ValueError(f"expected uint8 (N,H,W,3), got {rgb_u8.dtype} {tuple(rgb_u8.shape)}")
        rgb_u8 = rgb_u8.to(self.device).contiguous()
        n, h, w, _ = rgb_u8.shape
        if n == 0 or h == 0 or w == 0:
            res = {}
            if tensors:
                res.update({k: torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device) for k in ("x", "wb", "he", "gc")})
            if images:
                res.update({k: torch.empty((n, h, w, 3), dtype=torch.uint8, device=self.device) for k in ("wb_u8", "he_u8", "gc_u8")})
            return res
        res = {}
        ptr = {k: None for k in ("x", "wb", "he", "gc", "wb_u8", "he_u8", "gc_u8")}
        if tensors:
            for k in ("x", "wb", "he", "gc"):
                res[k] = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
                ptr[k] = res[k].data_ptr()
        if images:
            for k in ("wb_u8", "he_u8", "gc_u8"):
                res[k] = torch.empty((n, h, w, 3), dtype=torch.uint8, device=self.device)
                ptr[k] = res[k].data_ptr()
        ws = self._workspace("preprocess", self.lib.wn_preprocess_workspace_bytes(n, h, w))
        self._call("wn_preprocess_u8", rgb_u8.data_ptr(), n, h, w, ptr["x"], ptr["wb"], ptr["he"], ptr["gc"],
                   ptr["wb_u8"], ptr["he_u8"], ptr["gc_u8"], ws.data_ptr(), ws.numel())
        return res

    def white_balance_gray(self, gray_u8: torch.Tensor) -> torch.Tensor:
        """Grayscale branch of ``white_balance_transform`` (data.py:30-36) on uint8 (N,H,W) CUDA tensors."""
        if gray_u8.dtype != torch.uint8 or gray_u8.dim() != 3:
            raise ValueError(f"expected uint8 (N,H,W), got {gray_u8.dtype} {tuple(gray_u8.shape)}")
        g = gray_u8.to(self.device).contiguous()
        out = torch.empty_like(g)
        if g.numel() == 0:
            return out
        n, h, w = g.shape
        ws = self._workspace("preprocess", self.lib.wn_white_balance_gray_workspace_bytes(n, h, w))
        self._call("wn_white_balance_gray_u8", g.data_ptr(), out.data_ptr(), n, h, w, ws.data_ptr(), ws.numel())
        return out

    def resize_batch(self, images, dst_h: int, dst_w: int, swap_rb: bool = False) -> torch.Tensor:
        """Batched ``cv2.resize(img, (dst_w, dst_h))`` (+ optional BGR<->RGB swap) of differently sized uint8 HWC
        images (numpy arrays or CUDA tensors) into one uint8 (N, dst_h, dst_w, 3) CUDA tensor -- bit-exact
        OpenCV INTER_LINEAR arithmetic on the device (wn_resize_u8; training_utils.py:94-107)."""
        devs = []
        for im in images:
            t = torch.from_numpy(np.ascontiguousarray(im)) if isinstance(im, np.ndarray) else im
            if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
                raise ValueError(f"expected uint8 HWC images, got {t.dtype} {tuple(t.shape)}")
            devs.append(t.to(self.device, non_blocking=True).contiguous())
        n = len(devs)
        out = torch.empty((n, dst_h, dst_w, 3), dtype=torch.uint8, device=self.device)
        if n == 0 or out.numel() == 0:
            return out
        hs, ws = _sizes([t.shape[:2] for t in devs])
        self._call("wn_resize_u8", _ptrs(devs), hs, ws, n, out.data_ptr(), dst_h, dst_w, 1 if swap_rb else 0)
        for t in devs:  # the kernel reads them on the current stream after this call returns
            t.record_stream(torch.cuda.current_stream(self.device))
        return out

    def postprocess(self, out: torch.Tensor) -> torch.Tensor:
        """ten2arr on the device: fp32 (N,3,H,W) -> uint8 (N,H,W,3) CUDA tensor."""
        out = out.detach().to(self.device, torch.float32).contiguous()
        n, c, h, w = out.shape
        if c != 3:
            raise ValueError("expected (N,3,H,W)")
        res = torch.empty((n, h, w, 3), dtype=torch.uint8, device=self.device)
        if res.numel() == 0:
            return res
        self._call("wn_postprocess_u8", out.data_ptr(), res.data_ptr(), n, h, w)
        return res

    def _enhance_args(self, rgb_u8, out_u8, out_f32):
        if rgb_u8.dtype != torch.uint8 or rgb_u8.dim() != 4 or rgb_u8.shape[3] != 3:
            raise ValueError(f"expected uint8 (N,H,W,3), got {rgb_u8.dtype} {tuple(rgb_u8.shape)}")
        rgb_u8 = rgb_u8.to(self.device).contiguous()
        n, h, w, _ = rgb_u8.shape
        if out_u8 is None:
            out_u8 = torch.empty((n, h, w, 3), dtype=torch.uint8, device=self.device)
        elif (out_u8.dtype != torch.uint8 or tuple(out_u8.shape) != (n, h, w, 3) or not out_u8.is_contiguous()
              or out_u8.device != rgb_u8.device):
            raise ValueError(f"out_u8 must be a contiguous uint8 {(n, h, w, 3)} tensor on {rgb_u8.device}, got "
                             f"{out_u8.dtype} {tuple(out_u8.shape)} strides {out_u8.stride()} on {out_u8.device}")
        if out_f32 is not None and (out_f32.dtype != torch.float32 or tuple(out_f32.shape) != (n, 3, h, w)
                                    or not out_f32.is_contiguous() or out_f32.device != rgb_u8.device):
            raise ValueError(f"out_f32 must be a contiguous float32 {(n, 3, h, w)} tensor on {rgb_u8.device}")
        return rgb_u8, out_u8

    def enhance(self, rgb_u8: torch.Tensor, mode: int = _lib.MODE_DEFAULT, out_u8: Optional[torch.Tensor] = None,
                out_f32: Optional[torch.Tensor] = None, peer_out=()) -> torch.Tensor:
        """preprocess -> forward -> postprocess on uint8 (N,H,W,3) CUDA input; returns uint8 NHWC.

        ``peer_out``: device addresses (ints) inside other ranks' buffers (``dist.PeerGather.peer_addresses``) that
        receive the same bytes as ``out_u8`` from the kernel that writes it (wn_enhance_u8_peers)."""
        rgb_u8, out_u8 = self._enhance_args(rgb_u8, out_u8, out_f32)
        n, h, w, _ = rgb_u8.shape
        if out_u8.numel() == 0:
            return out_u8
        ws = self._workspace("enhance", self.lib.wn_enhance_workspace_bytes(n, h, w, mode))
        peers = (ctypes.c_void_p * max(1, len(peer_out)))(*peer_out)  # addresses, not tensors
        self._call("wn_enhance_u8_peers", rgb_u8.data_ptr(), out_u8.data_ptr(),
                   None if out_f32 is None else out_f32.data_ptr(), peers, len(peer_out), n, h, w, mode, ws.data_ptr(),
                   ws.numel())
        return out_u8

    DEFAULT_TILE = (998, 998)  # a window (tile + 13 pixels of context per side) of at most 1024 x 1024

    # ---- tile "auto": whole images where their workspace fits a budget, else windows of DEFAULT_TILE ----------------
    # The budget of auto_tile in bytes; None: half the device's total memory (42.5 GB on an H100 80GB).  It comes from
    # the card, not from its free memory, so that other work on a shared card never decides which path a call takes
    # (in training the two paths differ in the last bits of the gradients).
    AUTO_WORKSPACE_BYTES: Optional[int] = None

    @classmethod
    def whole_image_bytes(cls, kind: str, shapes, mode: int, train_mode: Optional[int] = None) -> int:
        """The device memory the whole-image path of one call of ``kind`` takes, from the library's workspace
        queries, or 0 where that path refuses the call.  ``shapes``: (n, h, w), or [(h, w), ...] for "ragged".

        Kinds: "net" (``WaterNet``), "cmg", "refiner" -- with ``train_mode`` None the inference workspace
        (wn_forward_workspace_bytes, wn_submodule_workspace_bytes: the largest pass), else the sum of the training
        workspaces of the slices ``_train_slices`` makes, all of which are kept until backward; "ragged"
        (``forward_many`` under autograd: the training calls of ``ragged_train_calls``); "enhance" (uint8,
        wn_enhance_workspace_bytes) and "vgg" (the perceptual loss with one window per image)."""
        lib = _lib.load()
        if kind == "ragged":
            sizes = [(h, w) for h, w in shapes if h * w > 0]
            if any(h * w > cls.TRAIN_MAX_PIXELS for h, w in sizes):
                return 0
            parts = [lib.wn_train_ragged_workspace_bytes(*_sizes([sizes[k] for k in idx]), len(idx))
                     for idx in ragged_train_calls(sizes, cls.TRAIN_MAX_PIXELS)]
            return 0 if 0 in parts else int(sum(parts))
        n, h, w = (int(v) for v in shapes)
        if kind == "enhance":
            return int(lib.wn_enhance_workspace_bytes(n, h, w, mode))
        if kind == "vgg":
            return int(lib.wn_perceptual_loss_workspace_bytes(n, h, w, 0, 0, 0))
        if kind not in ("net", "cmg", "refiner"):
            raise ValueError(f"unknown kind {kind!r}")
        if train_mode is None:
            query = lib.wn_forward_workspace_bytes if kind == "net" else lib.wn_submodule_workspace_bytes
            return int(query(n, h, w, mode))
        if n <= 0 or h * w > cls.TRAIN_MAX_PIXELS:
            return 0
        stack = cls.STACK_CMG if kind == "cmg" else cls.STACK_REFINER
        parts = [lib.wn_train_workspace_bytes(b - a, h, w) if kind == "net" else
                 lib.wn_submodule_train_workspace_bytes(b - a, h, w, stack)
                 for a, b in cls._train_slice_bounds(n, h, w)]
        return 0 if 0 in parts else int(sum(parts))

    @classmethod
    def auto_tile(cls, kind: str, shapes, mode: int, train_mode: Optional[int] = None, device=None):
        """What tile (or grad_tile) "auto" means for one call: None (whole images) when ``whole_image_bytes`` of the
        call is at most the budget (``AUTO_WORKSPACE_BYTES``, or half of ``device``'s memory), else DEFAULT_TILE.  A
        call the whole-image path refuses takes windows; a call without pixels and any call in ``mode``
        MODE_FP32_SIMT (which has no windowed path) take whole images."""
        sizes = shapes if kind == "ragged" else [tuple(shapes[1:])] if shapes[0] > 0 else []
        if mode == _lib.MODE_FP32_SIMT or not any(h * w for h, w in sizes):
            return None
        need = cls.whole_image_bytes(kind, shapes, mode, train_mode)
        budget = cls.AUTO_WORKSPACE_BYTES
        if budget is None:
            budget = torch.cuda.get_device_properties(_require_cuda(device)).total_memory // 2
        return None if 0 < need <= budget else cls.DEFAULT_TILE

    @staticmethod
    def _tile_hw(tile) -> Tuple[int, int]:
        th, tw = (tile, tile) if isinstance(tile, (int, np.integer)) else tuple(tile)
        if int(th) < 1 or int(tw) < 1:
            raise ValueError(f"tile must be at least 1 x 1, got {tile!r}")
        return int(th), int(tw)

    def tiled_workspace_bytes(self, n: int, h: int, w: int, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                              max_pass_pixels: int = 0) -> int:
        """Workspace of one ``enhance_tiled`` call (wn_enhance_tiled_workspace_bytes); 0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_enhance_tiled_workspace_bytes(n, h, w, th, tw, int(max_pass_pixels), mode))

    def enhance_tiled(self, rgb_u8: torch.Tensor, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                      out_u8: Optional[torch.Tensor] = None, out_f32: Optional[torch.Tensor] = None,
                      max_pass_pixels: int = 0) -> torch.Tensor:
        """``enhance`` computed in overlapping windows (wn_enhance_u8_tiled): the same bits, with a workspace that
        does not grow with the image size.  ``tile``: the largest output tile, an int or (h, w); ``max_pass_pixels``:
        window pixels per pass (0 = 8 Mi).  Tensor-core modes only."""
        th, tw = self._tile_hw(tile)
        rgb_u8, out_u8 = self._enhance_args(rgb_u8, out_u8, out_f32)
        n, h, w, _ = rgb_u8.shape
        if out_u8.numel() == 0:
            return out_u8
        nbytes = self.lib.wn_enhance_tiled_workspace_bytes(n, h, w, th, tw, int(max_pass_pixels), mode)
        ws = self._workspace("enhance", nbytes)
        self._call("wn_enhance_u8_tiled", rgb_u8.data_ptr(), out_u8.data_ptr(),
                   None if out_f32 is None else out_f32.data_ptr(), n, h, w, th, tw, int(max_pass_pixels), mode,
                   ws.data_ptr(), ws.numel())
        return out_u8

    # ---- the tiled forward of fp32 tensors (wn_forward_tiled, wn_confidence_maps_tiled, wn_refine_tiled) ----------
    def forward_tiled_workspace_bytes(self, n: int, h: int, w: int, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                                      max_pass_pixels: int = 0) -> int:
        """Workspace of one ``forward_tiled`` call (wn_forward_tiled_workspace_bytes); 0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_forward_tiled_workspace_bytes(n, h, w, th, tw, int(max_pass_pixels), mode))

    def submodule_tiled_workspace_bytes(self, n: int, h: int, w: int, tile=DEFAULT_TILE,
                                        mode: int = _lib.MODE_DEFAULT, max_pass_pixels: int = 0) -> int:
        """Workspace of one ``confidence_maps_tiled`` / ``refine_tiled`` call (wn_submodule_tiled_workspace_bytes);
        0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_submodule_tiled_workspace_bytes(n, h, w, th, tw, int(max_pass_pixels), mode))

    def forward_tiled(self, x, wb, he, gc, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                      out: Optional[torch.Tensor] = None, max_pass_pixels: int = 0) -> torch.Tensor:
        """``forward`` computed in overlapping windows (wn_forward_tiled): the same bits when every input value is an
        8-bit level or the untiled call runs the batch in one pass, with a workspace that does not grow with the
        image size.  ``tile`` and ``max_pass_pixels`` as in ``enhance_tiled``.  Tensor-core modes only."""
        th, tw = self._tile_hw(tile)
        ins = self._check_inputs((x, wb, he, gc))
        n, _, h, w = ins[0].shape
        if out is None:
            out = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
        elif (out.dtype != torch.float32 or tuple(out.shape) != (n, 3, h, w) or not out.is_contiguous()
              or out.device != self.device):
            raise ValueError(f"out must be a contiguous float32 {(n, 3, h, w)} tensor on {self.device}")
        if out.numel() == 0:
            return out
        ws = self._workspace("forward", self.forward_tiled_workspace_bytes(n, h, w, (th, tw), mode, max_pass_pixels))
        self._call("wn_forward_tiled", *(t.data_ptr() for t in ins), _strides(ins), out.data_ptr(), n, h, w, th, tw,
                   int(max_pass_pixels), mode, ws.data_ptr(), ws.numel())
        return out

    def confidence_maps_tiled(self, x, wb, he, gc, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                              max_pass_pixels: int = 0) -> torch.Tensor:
        """``confidence_maps`` computed in overlapping windows (wn_confidence_maps_tiled)."""
        th, tw = self._tile_hw(tile)
        ins = self._check_inputs((x, wb, he, gc))
        n, _, h, w = ins[0].shape
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
        if out.numel() == 0:
            return out
        ws = self._workspace("forward", self.submodule_tiled_workspace_bytes(n, h, w, (th, tw), mode, max_pass_pixels))
        self._call("wn_confidence_maps_tiled", *(t.data_ptr() for t in ins), _strides(ins), out.data_ptr(), n, h, w,
                   th, tw, int(max_pass_pixels), mode, ws.data_ptr(), ws.numel())
        return out

    def refine_tiled(self, which: int, x, xbar, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                     max_pass_pixels: int = 0) -> torch.Tensor:
        """``refine`` computed in overlapping windows (wn_refine_tiled)."""
        th, tw = self._tile_hw(tile)
        ins = self._check_inputs((x, xbar))
        n, _, h, w = ins[0].shape
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device)
        if out.numel() == 0:
            return out
        ws = self._workspace("forward", self.submodule_tiled_workspace_bytes(n, h, w, (th, tw), mode, max_pass_pixels))
        self._call("wn_refine_tiled", int(which), *(t.data_ptr() for t in ins), _strides(ins), out.data_ptr(), n, h,
                   w, th, tw, int(max_pass_pixels), mode, ws.data_ptr(), ws.numel())
        return out

    def ragged_workspace_bytes(self, sizes, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                               max_pass_pixels: int = 0) -> int:
        """Workspace of one ``enhance_ragged`` call over images of ``sizes`` [(h, w), ...]
        (wn_enhance_ragged_workspace_bytes); 0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_enhance_ragged_workspace_bytes(*_sizes(sizes), len(sizes), th, tw, int(max_pass_pixels),
                                                              mode))

    def enhance_ragged(self, images: Sequence[torch.Tensor], tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                       out_u8: Optional[Sequence[torch.Tensor]] = None,
                       out_f32: Optional[Sequence[Optional[torch.Tensor]]] = None,
                       max_pass_pixels: int = 0) -> list:
        """``enhance`` of n uint8 (H_i,W_i,3) CUDA images of their own sizes in one call (wn_enhance_u8_ragged).
        Each image's outputs equal, bit for bit, ``enhance`` of that image alone (while the e4m3 range guard stays
        down).  ``tile`` and ``max_pass_pixels`` as in ``enhance_tiled``.  ``out_u8`` / ``out_f32``: optional lists of
        per-image outputs, uint8 (H_i,W_i,3) and float32 (1,3,H_i,W_i); an ``out_f32`` entry may be None.  Returns the
        list of uint8 outputs.  Tensor-core modes only."""
        th, tw = self._tile_hw(tile)
        n = len(images)
        if out_u8 is not None and len(out_u8) != n or out_f32 is not None and len(out_f32) != n:
            raise ValueError(f"out_u8 / out_f32 must hold one entry per image ({n})")
        srcs, outs = [], []
        for i, img in enumerate(images):
            if img.dim() != 3:
                raise ValueError(f"image {i}: expected uint8 (H,W,3), got {img.dtype} {tuple(img.shape)}")
            src, dst = self._enhance_args(img[None], None if out_u8 is None else out_u8[i][None],
                                          None if out_f32 is None else out_f32[i])
            srcs.append(src[0])
            outs.append(dst[0] if out_u8 is None else out_u8[i])
        entries = []
        for i, (src, dst) in enumerate(zip(srcs, outs)):
            if src.numel() == 0:  # zero-pixel images: empty outputs, no library call
                continue
            f32 = None if out_f32 is None else out_f32[i]
            entries.append(_lib.RaggedImage(src.data_ptr(), dst.data_ptr(), None if f32 is None else f32.data_ptr(),
                                            src.shape[0], src.shape[1]))
        if not entries:
            return outs
        nbytes = self.ragged_workspace_bytes([(e.height, e.width) for e in entries], (th, tw), mode, max_pass_pixels)
        ws = self._workspace("enhance", nbytes)
        table = (_lib.RaggedImage * len(entries))(*entries)
        self._call("wn_enhance_u8_ragged", table, len(entries), th, tw, int(max_pass_pixels), mode, ws.data_ptr(),
                   ws.numel())
        return outs

    # ---- ragged batches of fp32 tensors (wn_forward_ragged, wn_forward_train_ragged / wn_backward_ragged) ---------
    def _ragged_items(self, items, outputs: bool = True):
        """items: [(x, wb, he, gc), ...], each four (N_i,3,H_i,W_i) tensors.  Returns the checked inputs, one
        contiguous output per item (None without ``outputs``) and the flat list of its images as (item, index in the
        item, h, w), zero-pixel images left out."""
        ins, outs, images = [], [], []
        for i, item in enumerate(items):
            if len(item) != 4:
                raise ValueError(f"item {i}: expected the four tensors (x, wb, he, gc), got {len(item)}")
            t = self._check_inputs(item)
            n, _, h, w = t[0].shape
            ins.append(t)
            outs.append(torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device) if outputs else None)
            if h * w > 0:
                images += [(i, j, h, w) for j in range(n)]
        return ins, outs, images

    @staticmethod
    def _ragged_tensors(ins, outs, images):
        """wn_ragged_tensors descriptors of ``images`` (as ``_ragged_items`` lists them)."""
        table = (_lib.RaggedTensors * len(images))()
        for k, (i, j, h, w) in enumerate(images):
            t = ins[i]
            d = table[k]
            d.x, d.wb, d.he, d.gc = (u[j].data_ptr() for u in t)
            d.in_strides[:] = [s for u in t for s in u.stride()]
            d.out = outs[i][j].data_ptr() if outs[i] is not None else None
            d.height, d.width = h, w
        return table

    @staticmethod
    def _ragged_input_grads(gin, images):
        """input_grads_host of the ragged backward calls: the four input gradients of each of ``images`` (as
        ``_ragged_items`` lists them) from ``gin`` (per item, four tensors or None), or None when none is asked for."""
        if all(t is None for row in gin for t in row):
            return None
        return _ptrs([None if gin[i][t] is None else gin[i][t][j] for i, j, _, _ in images for t in range(4)])

    def forward_ragged_workspace_bytes(self, sizes, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT,
                                       max_pass_pixels: int = 0) -> int:
        """Workspace of one ``forward_ragged`` call over images of ``sizes`` [(h, w), ...]
        (wn_forward_ragged_workspace_bytes); 0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_forward_ragged_workspace_bytes(*_sizes(sizes), len(sizes), th, tw, int(max_pass_pixels),
                                                              mode))

    def forward_ragged(self, items, tile=DEFAULT_TILE, mode: int = _lib.MODE_DEFAULT, max_pass_pixels: int = 0) -> list:
        """``forward`` of images of their own sizes in one call (wn_forward_ragged).  ``items``: a list of 4-tuples
        (x, wb, he, gc) of (N_i,3,H_i,W_i) CUDA tensors of any strides; every image of every item is one entry of the
        ragged batch.  Returns one contiguous (N_i,3,H_i,W_i) output per item, each image bit for bit what ``forward``
        returns for it alone (while the e4m3 range guard stays down).  ``tile`` and ``max_pass_pixels`` as in
        ``enhance_ragged``.  Tensor-core modes only."""
        th, tw = self._tile_hw(tile)
        ins, outs, images = self._ragged_items(items)
        if not images:
            return outs
        nbytes = self.forward_ragged_workspace_bytes([(h, w) for _, _, h, w in images], (th, tw), mode,
                                                     max_pass_pixels)
        ws = self._workspace("forward", nbytes)
        self._call("wn_forward_ragged", self._ragged_tensors(ins, outs, images), len(images), th, tw,
                   int(max_pass_pixels), mode, ws.data_ptr(), ws.numel())
        return outs

    def _train_ragged_workspace(self, nbytes: int) -> torch.Tensor:
        """One training call's own workspace (it lives until backward), or that of one backward_ragged_tiled call."""
        return torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)

    def forward_train_ragged(self, items, train_mode: int = _lib.MODE_BF16X3):
        """``forward_train`` of images of their own sizes (wn_forward_train_ragged): ``items`` as ``forward_ragged``.
        The images are grouped into training calls by ``ragged_train_calls``; each call runs its images as one pass
        of equally sized slots and keeps the activations in its own workspace.  Returns (one output per item, saved
        state for ``backward_ragged``).  Each image's output equals ``forward_train`` of that image alone bit for
        bit.  One image over TRAIN_MAX_PIXELS is refused."""
        ins, outs, images = self._ragged_items(items)
        self.set_train_mode(train_mode)
        for i, j, h, w in images:
            if h * w > self.TRAIN_MAX_PIXELS:
                raise _lib.WaterNetLibraryError(
                    f"item {i}: one {h}x{w} image exceeds the {self.TRAIN_MAX_PIXELS >> 20} Mi pixels of one training "
                    "call; set WaterNet.grad_tile to train it in overlapping windows (wn_backward_tiled)")
        calls = []
        for idx in ragged_train_calls([(h, w) for _, _, h, w in images], self.TRAIN_MAX_PIXELS):
            imgs = [images[k] for k in idx]
            hs, wss = _sizes([(h, w) for _, _, h, w in imgs])
            ws = self._train_ragged_workspace(self.lib.wn_train_ragged_workspace_bytes(hs, wss, len(imgs)))
            self._call("wn_forward_train_ragged", self._ragged_tensors(ins, outs, imgs), len(imgs), ws.data_ptr(),
                       ws.numel())
            calls.append((imgs, hs, wss, ws))
        return outs, calls

    def backward_ragged(self, grad_outs, saved, shapes, want_inputs=None, train_mode: int = _lib.MODE_BF16X3):
        """d(loss)/d(out) of every item (a list of (N_i,3,H_i,W_i) tensors) + the state of ``forward_train_ragged``
        -> the 34 parameter gradients (state-dict order), the gradients of all images summed call by call in call
        order, and one list of four input gradients per item (None where ``want_inputs[i][t]`` is false, or
        everywhere when ``want_inputs`` is None)."""
        self.set_train_mode(train_mode)
        grads_out = [g.detach().to(self.device, torch.float32).contiguous() for g in grad_outs]
        gin = self._ragged_gin(grads_out, want_inputs)

        def run(call, dst):
            imgs, hs, wss, ws = call
            self._call("wn_backward_ragged", hs, wss, _ptrs([grads_out[i][j] for i, j, _, _ in imgs]),
                       _grads_array(dst), self._ragged_input_grads(gin, imgs), len(imgs), ws.data_ptr(), ws.numel())
        return self._sum_in_order(shapes, saved or [], run), gin

    @staticmethod
    def _ragged_gin(grads_out, want_inputs):
        """The input gradients of the ragged backward calls: per item, four tensors like its output gradient, None
        where ``want_inputs[i][t]`` is false or everywhere when ``want_inputs`` is None.  Every image with pixels is
        written whole by the library; zero-pixel items have no elements."""
        return [[torch.empty_like(g) if want_inputs is not None and want_inputs[i][t] else None for t in range(4)]
                for i, g in enumerate(grads_out)]

    # ---- windowed recompute backward (wn_backward_tiled) -------------------------------------------
    def backward_tiled_workspace_bytes(self, n: int, h: int, w: int, tile=DEFAULT_TILE, max_pass_pixels: int = 0) -> int:
        """Workspace of one ``backward_tiled`` call (wn_backward_tiled_workspace_bytes); 0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_backward_tiled_workspace_bytes(n, h, w, th, tw, int(max_pass_pixels)))

    def backward_tiled(self, grad_out: torch.Tensor, inputs, shapes, tile=DEFAULT_TILE, want_input_grads: bool = False,
                       max_pass_pixels: int = 0, train_mode: int = _lib.MODE_BF16X3):
        """The gradients of ``backward`` from the four input images alone (wn_backward_tiled): the training forward
        is recomputed in the overlapping windows of ``forward_tiled``, one pass of windows at a time, so no
        activation outlives the call and the workspace does not grow with the image size.  ``max_pass_pixels``:
        window pixels per pass (0 = 2 Mi, ~11.8 GB).  The workspace is allocated for this call only.  ``train_mode``:
        the arithmetic of the recomputed forward and of the backward."""
        grads, gin = self._windowed_backward("wn_backward_tiled", (), None, 0, "grad_out", grad_out, inputs, shapes,
                                             tile, (want_input_grads,) * 4, max_pass_pixels, train_mode)
        return (grads, gin) if want_input_grads else grads

    def _windowed_backward(self, what: str, lead, stack, first: int, grad_name: str, grad, inputs, shapes, tile,
                           want_inputs, max_pass_pixels, train_mode: int):
        """One call of ``what`` (``lead`` before the inputs) that recomputes the training forward of ``inputs`` in
        windows, with a workspace of its own (of the whole network for ``stack`` None, else of that stack): the
        parameter gradients of ``shapes`` (state-dict entries first, first + 1, ...) and the input gradients asked for
        by ``want_inputs`` (None where not).  An empty batch has zero gradients and makes no call."""
        self.set_train_mode(train_mode)
        th, tw = self._tile_hw(tile)
        ins = self._check_inputs(inputs)
        g = grad.detach().to(self.device, torch.float32).contiguous()
        n, _, h, w = ins[0].shape
        if tuple(g.shape) != (n, 3, h, w):
            raise ValueError(f"{grad_name} must be {(n, 3, h, w)}, got {tuple(g.shape)}")
        grads = self._param_grads(shapes, g.numel() > 0)
        make = torch.empty if g.numel() else torch.zeros
        gin = [make((n, 3, h, w), dtype=torch.float32, device=self.device) if want else None for want in want_inputs]
        if g.numel() == 0:
            return grads, gin
        nbytes = _require_workspace(
            self.backward_tiled_workspace_bytes(n, h, w, (th, tw), max_pass_pixels) if stack is None else
            self.submodule_backward_tiled_workspace_bytes(n, h, w, stack, (th, tw), max_pass_pixels),
            f"{what} rejects n={n} h={h} w={w} tile={th}x{tw} max_pass_pixels={max_pass_pixels}")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self._call(what, *lead, *(t.data_ptr() for t in ins), _strides(ins), g.data_ptr(), _grads_array(grads, first),
                   _ptrs(gin) if any(want_inputs) else None, n, h, w, th, tw, int(max_pass_pixels), ws.data_ptr(),
                   ws.numel())
        return grads, gin

    # ---- windowed recompute backward of a ragged batch (wn_backward_ragged_tiled) -------------------------------
    def backward_ragged_tiled_workspace_bytes(self, sizes, tile=DEFAULT_TILE, max_pass_pixels: int = 0) -> int:
        """Workspace of one ``backward_ragged_tiled`` call over images of ``sizes`` [(h, w), ...]
        (wn_backward_ragged_tiled_workspace_bytes); 0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_backward_ragged_tiled_workspace_bytes(*_sizes(sizes), len(sizes), th, tw,
                                                                     int(max_pass_pixels)))

    def backward_ragged_tiled(self, grad_outs, items, shapes, tile=DEFAULT_TILE, want_inputs=None,
                              max_pass_pixels: int = 0, train_mode: int = _lib.MODE_BF16X3):
        """The gradients of ``backward_ragged`` from the input images alone (wn_backward_ragged_tiled): ``items`` as
        ``forward_ragged`` takes them, ``grad_outs`` one (N_i,3,H_i,W_i) tensor per item.  The windows of ``tile`` of
        every image are packed into passes of ``max_pass_pixels`` slot pixels (0 = 2 Mi), and the training forward
        is recomputed one pass at a time, so no activation outlives the call.  Returns the 34 parameter gradients
        (state-dict order, summed over the images) and one list of four input gradients per item (None where
        ``want_inputs[i][t]`` is false, or everywhere when ``want_inputs`` is None).  Zero-pixel items get zero
        gradients.  The workspace is allocated for this call only.  ``train_mode`` as ``backward_tiled``."""
        self.set_train_mode(train_mode)
        th, tw = self._tile_hw(tile)
        ins, _, images = self._ragged_items(items, outputs=False)
        grads_out = [g.detach().to(self.device, torch.float32).contiguous() for g in grad_outs]
        for i, (t, g) in enumerate(zip(ins, grads_out)):
            if g.shape != t[0].shape:
                raise ValueError(f"item {i}: the output gradient must be {tuple(t[0].shape)}, got {tuple(g.shape)}")
        grads = self._param_grads(shapes, bool(images))
        gin = self._ragged_gin(grads_out, want_inputs)
        if not images:
            return grads, gin
        sizes = [(h, w) for _, _, h, w in images]
        nbytes = _require_workspace(
            self.backward_ragged_tiled_workspace_bytes(sizes, (th, tw), max_pass_pixels),
            f"wn_backward_ragged_tiled rejects {len(images)} images up to {max(h for h, _ in sizes)}x"
            f"{max(w for _, w in sizes)} at tile={th}x{tw} max_pass_pixels={max_pass_pixels}")
        ws = self._train_ragged_workspace(nbytes)
        self._call("wn_backward_ragged_tiled", self._ragged_tensors(ins, [None] * len(ins), images),
                   _ptrs([grads_out[i][j] for i, j, _, _ in images]), _grads_array(grads),
                   self._ragged_input_grads(gin, images), len(images), th, tw, int(max_pass_pixels), ws.data_ptr(),
                   ws.numel())
        return grads, gin

    # ---- windowed recompute backward of one sub-module (wn_confidence_maps_backward_tiled, wn_refine_backward_tiled) --
    def submodule_backward_tiled_workspace_bytes(self, n: int, h: int, w: int, stack: int, tile=DEFAULT_TILE,
                                                 max_pass_pixels: int = 0) -> int:
        """Workspace of one ``confidence_maps_backward_tiled`` (stack 0) or ``refine_backward_tiled`` (stack 1) call
        (wn_submodule_backward_tiled_workspace_bytes); 0 for rejected arguments."""
        th, tw = self._tile_hw(tile)
        return int(self.lib.wn_submodule_backward_tiled_workspace_bytes(n, h, w, th, tw, int(max_pass_pixels),
                                                                        int(stack)))

    def confidence_maps_backward_tiled(self, grad_maps, inputs, shapes, tile=DEFAULT_TILE, want_inputs=(False,) * 4,
                                       max_pass_pixels: int = 0, train_mode: int = _lib.MODE_BF16X3):
        """The gradients of ``confidence_maps_backward`` from the four input images alone
        (wn_confidence_maps_backward_tiled): the cmg's training forward is recomputed in the overlapping windows of
        ``confidence_maps_tiled``, one pass at a time, so no activation outlives the call and the workspace does not
        grow with the image size.  ``max_pass_pixels``: window pixels per pass (0 = 2 Mi, ~8.1 GB).  Returns the 16
        parameter gradients and the input gradients ``want_inputs`` asks for (else None).  The workspace is allocated
        for this call only."""
        ins = self._check_inputs(inputs)  # a sub-module call reports bad inputs before a bad tile or mode
        return self._windowed_backward("wn_confidence_maps_backward_tiled", (), self.STACK_CMG, 0,
                                       "the output gradient", grad_maps, ins, shapes, tile, want_inputs,
                                       int(max_pass_pixels), train_mode)

    def refine_backward_tiled(self, which: int, grad_out, inputs, shapes, tile=DEFAULT_TILE,
                              want_inputs=(False, False), max_pass_pixels: int = 0, train_mode: int = _lib.MODE_BF16X3):
        """The gradients of ``refine_backward`` from x and xbar alone (wn_refine_backward_tiled), as
        ``confidence_maps_backward_tiled`` (0 = 2 Mi window pixels per pass, ~3.8 GB)."""
        ins = self._check_inputs(inputs)
        return self._windowed_backward("wn_refine_backward_tiled", (int(which),), self.STACK_REFINER,
                                       16 + 6 * int(which), "the output gradient", grad_out, ins, shapes, tile,
                                       want_inputs, int(max_pass_pixels), train_mode)

    # ---- the VGG19 perceptual loss (wn_perceptual_loss) ----------------------------------------
    def pack_vgg_weights(self, params: Sequence[torch.Tensor], key=None) -> None:
        """params: weight and bias of VGG19's 16 convolutions in ``features`` order (32 tensors).  Skipped when
        ``key`` equals the key of the last pack."""
        if len(params) != _lib.VGG_NUM_PARAMS:
            raise ValueError(f"expected {_lib.VGG_NUM_PARAMS} VGG parameter tensors, got {len(params)}")
        for i, (cin, cout) in enumerate(VGG_CONVS):  # the kernels read these shapes: anything else is refused
            want = ((cout, cin, 3, 3), (cout,))
            got = (tuple(params[2 * i].shape), tuple(params[2 * i + 1].shape))
            if got != want:
                raise ValueError(f"VGG convolution {i}: weight and bias of shapes {got}, expected {want} (VGG19)")
        if key is not None and key == getattr(self, "_vgg_key", None):
            return
        staged = [p.detach().to(device=self.device, dtype=torch.float32).contiguous() for p in params]
        self._call("wn_vgg_pack_weights", _ptrs(staged))
        self._vgg_keepalive = staged  # until the async pack kernels have consumed them
        self._vgg_key = key

    def perceptual_loss_workspace_bytes(self, n: int, h: int, w: int, tile=None, max_pass_pixels: int = 0) -> int:
        th, tw = vgg_tile_hw(tile)
        return int(self.lib.wn_perceptual_loss_workspace_bytes(n, h, w, th, tw, int(max_pass_pixels)))

    def _vgg_workspace(self, n, h, w, th, tw, mpp, what):
        nbytes = int(self.lib.wn_perceptual_loss_workspace_bytes(n, h, w, th, tw, mpp))
        if nbytes == 0:
            hint = " (pass a tile)" if th == 0 and h * w > VGG_MAX_PIXELS else ""
            raise ValueError(f"{what}: unsupported arguments n={n} {h}x{w} tile={th}x{tw} max_pass_pixels={mpp}: images "
                             f"must be at least 16 x 16 and a window at most {VGG_MAX_PIXELS} pixels{hint}")
        return self._workspace("vgg", nbytes)

    def perceptual_loss(self, out, ref, tile=None, want_grad: bool = False, max_pass_pixels: int = 0,
                        train_mode: int = _lib.MODE_BF16X3):
        """mean((255 (F(out) - F(ref)))^2) with F = VGG19 features[:-1] of the normalised images, on the packed VGG
        weights (wn_perceptual_loss), in windows that own ``tile`` input pixels of features (None: one window per
        image).  Returns (0-d loss, d(loss)/d(out) as a contiguous (N,3,H,W) tensor, or None without ``want_grad``).
        ``train_mode``: the arithmetic of the VGG convolutions, MODE_BF16X3 or single-pass MODE_BF16."""
        self.set_train_mode(train_mode)
        o, r = (t.detach() if t.dtype == torch.float32 else t.detach().float() for t in (out, ref))
        for t in (o, r):
            if t.device != self.device or t.dim() != 4 or t.shape[1] != 3:
                raise ValueError(f"expected (N,3,H,W) inputs on {self.device}, got {tuple(t.shape)} on {t.device}")
        if o.shape != r.shape:
            raise ValueError(f"out and ref differ in shape: {tuple(o.shape)} vs {tuple(r.shape)}")
        n, _, h, w = o.shape
        th, tw = vgg_tile_hw(tile)
        mpp = int(max_pass_pixels)
        ws = self._vgg_workspace(n, h, w, th, tw, mpp, "perceptual_loss")
        loss = torch.empty((), dtype=torch.float32, device=self.device)
        grad = torch.empty((n, 3, h, w), dtype=torch.float32, device=self.device) if want_grad else None
        self._call("wn_perceptual_loss", o.data_ptr(), _strides((o,)), r.data_ptr(), _strides((r,)), n, h, w, th, tw,
                   mpp, loss.data_ptr(), grad.data_ptr() if grad is not None else None, ws.data_ptr(), ws.numel())
        return loss, grad

    def debug_vgg_layer(self, x, layer: int, tile=None, ref=None, train_mode: int = _lib.MODE_BF16X3) -> torch.Tensor:
        """Test aid (wn_debug_vgg_layer), as fp32 (N, C, H >> level, W >> level): launch ``layer`` (0..19) of the VGG
        forward of whole images; (20) the conv5_4 features of the windowed call with ``tile``; for the loss of
        (out = x, ``ref``): (21) the seed, d(loss)/d(conv5_4 before its ReLU); (22 + k) the output of the backward
        launch of forward launch k, d(loss)/d(input of launch k) (k = 0: 16 normalised channels, 3 real).
        ``train_mode`` as ``perceptual_loss``."""
        self.set_train_mode(train_mode)
        x = x.detach().float()
        n, _, h, w = x.shape
        th, tw = vgg_tile_hw(tile)
        steps = len(VGG_STEPS)
        if layer == steps:
            shape = (n, 512, h // 16, w // 16)
        elif layer == steps + 1:
            shape = (n, 512, h >> 4, w >> 4)
        elif layer > steps + 1:
            k = layer - steps - 2
            lv, ch = (VGG_STEPS[k - 1][1], VGG_STEPS[k - 1][2]) if k else (0, 16)
            shape = (n, ch, h >> lv, w >> lv)
        else:
            _, lv, ch = VGG_STEPS[layer]
            shape = (n, ch, h >> lv, w >> lv)
        r = ref.detach().float() if ref is not None else None
        dst = torch.empty(shape, dtype=torch.float32, device=self.device)
        ws = self._vgg_workspace(n, h, w, th, tw, 0, "debug_vgg_layer")
        self._call("wn_debug_vgg_layer", x.data_ptr(), _strides((x,)), r.data_ptr() if r is not None else None,
                   _strides((r,)) if r is not None else None, n, h, w, th, tw, int(layer), dst.data_ptr(),
                   ws.data_ptr(), ws.numel())
        return dst

    # ---- SSIM / PSNR statistics (wn_quality) ------------------------------------------------------------------
    def _check_pairs(self, outs, refs, groups) -> None:
        """ValueError unless outs and refs are as many (at least one) fp32 contiguous (3,H,W) tensors on this
        engine's device, pairwise of one shape, with one group each."""
        n = len(outs)
        if n == 0 or len(refs) != n or len(groups) != n:
            raise ValueError(f"expected as many refs and groups as outs (at least one), got {n}, {len(refs)}, "
                             f"{len(groups)}")
        for o, r in zip(outs, refs):
            for t in (o, r):
                if t.device != self.device or t.dtype != torch.float32 or t.dim() != 3 or t.shape[0] != 3 or \
                        not t.is_contiguous():
                    raise ValueError(f"expected fp32 contiguous (3,H,W) tensors on {self.device}, got "
                                     f"{t.dtype} {tuple(t.shape)} on {t.device}")
            if o.shape != r.shape:
                raise ValueError(f"out and ref differ in shape: {tuple(o.shape)} vs {tuple(r.shape)}")

    def quality_workspace_bytes(self, sizes) -> int:
        """Workspace of one ``quality`` call over images of ``sizes`` [(h, w), ...]; 0 for rejected sizes."""
        return int(self.lib.wn_quality_workspace_bytes(*_sizes(sizes), len(sizes)))

    def quality(self, outs, refs, groups) -> torch.Tensor:
        """The SSIM / PSNR statistics of the pairs (outs[i], refs[i]) in one wn_quality call: (3,H_i,W_i) fp32
        contiguous CUDA tensors, image i in group ``groups[i]`` (images of one group share SSIM's data range).
        Returns a (n, 7) float64 tensor, per image: the SSIM sum over its counted pixels, their count, the sum of
        squared differences, min and max of out, min and max of ref."""
        self._check_pairs(outs, refs, groups)
        n = len(outs)
        table = (_lib.QualityImage * n)()
        for d, o, r, g in zip(table, outs, refs, groups):
            d.out, d.ref, d.height, d.width, d.group = o.data_ptr(), r.data_ptr(), o.shape[1], o.shape[2], int(g)
        sizes = [tuple(o.shape[1:]) for o in outs]
        ws = self._workspace("quality", _require_workspace(
            self.quality_workspace_bytes(sizes), f"quality: unsupported sizes {sizes}: 1..65535 images, each side at "
                                                 "least 6 and at most 0x7fffffff / 3 pixels per plane"))
        stats = torch.empty((n, _lib.QUALITY_STATS), dtype=torch.float64, device=self.device)
        self._call("wn_quality", table, n, stats.data_ptr(), ws.data_ptr(), ws.numel())
        return stats

    # ---- SSIM's gradient (wn_ssim_grad) -------------------------------------------------------------------------
    def ssim_grad_workspace_bytes(self, sizes) -> int:
        """Workspace of one ``ssim_grad`` call over images of ``sizes`` [(h, w), ...]; 0 for rejected sizes."""
        return int(self.lib.wn_ssim_grad_workspace_bytes(*_sizes(sizes), len(sizes)))

    def ssim_grad(self, outs, refs, groups, scales, grads=None):
        """``quality``'s statistics of the pairs (outs[i], refs[i]) and, per image, d/d(outs[i]) of
        sum_j scales[j] * SSIM_j (SSIM_j: image j's SSIM, its data-range term included) in one wn_ssim_grad call.
        ``grads``: the (3,H_i,W_i) fp32 contiguous tensors that receive the gradients, None to allocate them; none
        may overlap an out, a ref or another grad.  Returns (stats, grads)."""
        self._check_pairs(outs, refs, groups)
        n = len(outs)
        if len(scales) != n:
            raise ValueError(f"expected one scale per image, got {len(scales)} for {n}")
        if grads is None:
            grads = [torch.empty_like(o) for o in outs]
        if len(grads) != n:
            raise ValueError(f"expected one grad per image, got {len(grads)} for {n}")
        for o, g in zip(outs, grads):
            if g.device != self.device or g.dtype != torch.float32 or g.shape != o.shape or not g.is_contiguous():
                raise ValueError(f"expected fp32 contiguous {tuple(o.shape)} grads on {self.device}, got {g.dtype} "
                                 f"{tuple(g.shape)} on {g.device}")
        table = (_lib.SSIMGradImage * n)()
        for d, o, r, g, grp, sc in zip(table, outs, refs, grads, groups, scales):
            d.out, d.ref, d.grad, d.height, d.width = o.data_ptr(), r.data_ptr(), g.data_ptr(), o.shape[1], o.shape[2]
            d.group, d.scale = int(grp), float(sc)
        sizes = [tuple(o.shape[1:]) for o in outs]
        ws = self._workspace("ssim_grad", _require_workspace(
            self.ssim_grad_workspace_bytes(sizes), f"ssim_grad: unsupported sizes {sizes}: 1..65535 images, each "
                                                   "side at least 6 and at most 0x7fffffff / 3 pixels per plane"))
        stats = torch.empty((n, _lib.QUALITY_STATS), dtype=torch.float64, device=self.device)
        self._call("wn_ssim_grad", table, n, stats.data_ptr(), ws.data_ptr(), ws.numel())
        return stats, grads
