"""WaterNet as an ``nn.Module`` whose forward runs on the CUDA kernels.

Mirror of the reference's ``waternet/net.py`` public surface (class names,
submodule and parameter names, forward signature and argument order) so that the
reference's checkpoints load with strict ``load_state_dict`` and callers
(``hubconf.py:75``, ``inference.py:88,191``, ``train.py:241,108``) do not change.

* ``WaterNet.forward(x, wb, ce, gc)`` (reference ``net.py:99-108``) dispatches to
  ``libwaternet_b200.so`` (``wn_forward``).  There is no CPU path: CPU tensors
  raise.
* When autograd needs a graph (training, ``train.py:100-133``), forward values and
  the 34 parameter gradients both come from the CUDA library (``wn_forward_train`` /
  ``wn_backward``: tensor-core data-gradient and weight-gradient kernels), including
  gradients of the input images when they require grad.  Only the fp32 CUDA-core mode
  re-evaluates the network with torch ops for its backward pass.
* The sub-modules (``model.cmg``, the refiners, free-standing instances) train on the library
  the same way (``wn_confidence_maps_train`` / ``wn_refine_train`` and their backward), with
  gradients for their own parameters and inputs only; with ``grad_tile`` set their gradients are recomputed in
  overlapping windows (``wn_confidence_maps_backward_tiled`` / ``wn_refine_backward_tiled``).
"""
from __future__ import annotations

import threading
import weakref
from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .engine import TRAIN_PASS_PIXELS, Engine, new_engine

MODES = {"default": _lib.MODE_DEFAULT, "fp32": _lib.MODE_FP32_SIMT, "bf16x3": _lib.MODE_BF16X3,
         "bf16_fp8": _lib.MODE_BF16_FP8}
# the arithmetic of the native training calls (wn_set_train_mode): three bf16 products per product (~1e-5 of fp32),
# or one (operands rounded to bf16 once, fp32 accumulation, as autocast trains convolutions)
TRAIN_PRECISIONS = {"bf16x3": _lib.MODE_BF16X3, "bf16": _lib.MODE_BF16}


def _checked_train_mode(train_precision) -> int:
    if train_precision not in TRAIN_PRECISIONS:
        raise ValueError(f"unknown train_precision {train_precision!r}; choose from {sorted(TRAIN_PRECISIONS)}")
    return TRAIN_PRECISIONS[train_precision]

# model -> {device index: Engine}.  Every module that can be called on its own (WaterNet and, like in the
# reference, its sub-modules) has a private engine per device = its own packed-weight slot in the library.
# Kept outside the module so that copy.deepcopy / pickling of a model never touches a C handle.
_model_engines = weakref.WeakKeyDictionary()
_model_engines_lock = threading.Lock()


def _checked_tile(tile, mode: int):
    """``tile`` as (h, w), or None for whole images per pass.  The tiled forward runs on the tensor cores only."""
    if tile is None:
        return None
    if mode == _lib.MODE_FP32_SIMT:
        raise ValueError("tile: the tiled forward runs on the tensor cores only, and precision='fp32' is the CUDA-core "
                         "mode; use precision='default' or 'bf16x3', or tile=None")
    return Engine._tile_hw(tile)


def _checked_grad_tile(grad_tile, mode: int):
    """``grad_tile`` as (h, w), or None for the untiled training path.  The windowed backward is tensor-core only."""
    if grad_tile is None:
        return None
    if mode == _lib.MODE_FP32_SIMT:
        raise ValueError("grad_tile: the windowed backward runs on the tensor cores only, and precision='fp32' is the "
                         "CUDA-core mode; use precision='default' or 'bf16x3', or grad_tile=None")
    return Engine._tile_hw(grad_tile)


def _param_version(p) -> int:
    try:
        return p._version
    except RuntimeError:  # tensors created under torch.inference_mode() do not track versions
        return -1


class _PackedWeightsMixin:
    """Packed-weight cache of a callable module.

    The kernels consume re-packed copies of the 34 tensors (``wn_pack_weights``).  The cache key is
    ``(data_ptr, _version)`` of every parameter plus an epoch that ``load_state_dict``, ``.to()/.cuda()/.float()``
    (``_apply``) and :meth:`invalidate_packed_weights` advance.  In-place updates through autograd-visible ops
    (optimizer steps, ``p.copy_()``, ``p.mul_()``) bump ``_version`` and are picked up automatically; writes through
    ``p.data`` (``p.data.copy_(ema)``) are invisible to ``_version`` -- call ``invalidate_packed_weights()`` after them.
    """

    def invalidate_packed_weights(self) -> None:
        object.__setattr__(self, "_pack_epoch", getattr(self, "_pack_epoch", 0) + 1)
        for child in self.children():
            if isinstance(child, _PackedWeightsMixin):
                child.invalidate_packed_weights()

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self.invalidate_packed_weights()
        return out

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        self.invalidate_packed_weights()
        return out

    def _engine_for(self, x, params, key_params=None):
        """This module's private engine on x's device with ``params`` (34 tensors, state-dict order) packed.  The
        cache key is taken over ``key_params`` when given (a free-standing stack: its own parameters, not the zeros
        that fill the other slots)."""
        if not x.is_cuda:
            raise _lib.WaterNetLibraryError(
                f"{type(self).__name__}.forward got CPU tensors: waternet_b200 has no CPU path; move the model and "
                "inputs to a CUDA device (H100)")
        if params[0].device != x.device:
            raise RuntimeError(f"model parameters on {params[0].device}, inputs on {x.device}")
        with _model_engines_lock:
            per_dev = _model_engines.setdefault(self, {})
            eng = per_dev.get(x.device.index)
            if eng is None:
                eng = per_dev[x.device.index] = new_engine(x.device)
        key = (getattr(self, "_pack_epoch", 0),) + tuple((p.data_ptr(), _param_version(p))
                                                         for p in (params if key_params is None else key_params))
        eng.pack_weights(params, key=key)
        return eng

# (in, out, kernel) of the confidence-map stack (reference net.py:12-42) and of a refiner (net.py:62-70)
CMG_SPEC = [(12, 128, 7), (128, 128, 5), (128, 128, 3), (128, 64, 1), (64, 64, 7), (64, 64, 5), (64, 64, 3), (64, 3, 3)]
REFINER_SPEC = [(6, 32, 7), (32, 32, 5), (32, 3, 3)]


def _same_conv(cin: int, cout: int, k: int) -> nn.Conv2d:
    return nn.Conv2d(cin, cout, kernel_size=k, stride=1, dilation=1, padding=k // 2)


class _ConvStack(_PackedWeightsMixin, nn.Module):
    """conv1..convK attributes (the names the reference's state dict uses).

    Like the reference's sub-modules (``net.py:45-56``, ``:75-80``) a stack can be called on its own.  Inside a
    ``WaterNet`` it runs with the parent's packed state dict (``wn_confidence_maps`` / ``wn_refine``); a
    free-standing instance packs its own tensors into the state-dict slots of its kind, zeros elsewhere.
    With autograd recording (a parameter or an input requires grad) a call on CUDA tensors in a tensor-core
    precision trains natively: the forward runs in the bf16x3 arithmetic of training and keeps the stack's
    activations (``wn_confidence_maps_train`` / ``wn_refine_train``), and backward gives the gradients of the stack's
    own parameters and of its inputs (``wn_confidence_maps_backward`` / ``wn_refine_backward``), in the arithmetic of
    ``train_precision`` (as ``WaterNet.train_precision``; the default "bf16x3").  Nothing reaches the
    parent's other parameters.  Whole images per call (``tile`` does not apply), at most ``Engine.TRAIN_MAX_PIXELS``
    pixels per image; a batch over that runs in slices.  CPU tensors, ``precision="fp32"`` and a larger image
    evaluate the torch graph instead.
    With ``grad_tile`` set (as ``WaterNet.grad_tile``) such a call keeps only its inputs: the forward is
    ``wn_confidence_maps_tiled`` / ``wn_refine_tiled`` in the bf16x3 arithmetic of training, and backward recomputes
    the stack's activations window by window (``wn_confidence_maps_backward_tiled`` / ``wn_refine_backward_tiled``),
    in about 8 GB for the cmg and 4 GB for a refiner whatever the image or batch size, with no limit on the image
    size.  Bound to a ``WaterNet`` a stack follows the parent's ``precision``, ``train_precision``, ``tile`` and
    ``grad_tile``; a free-standing one uses its own attributes.
    """

    spec: List[tuple] = []
    precision = "default"
    train_precision = "bf16x3"
    tile = None
    grad_tile = None

    def __init__(self):
        super().__init__()
        for i, (cin, cout, k) in enumerate(self.spec, start=1):
            setattr(self, f"conv{i}", _same_conv(cin, cout, k))
        object.__setattr__(self, "_parent_ref", None)   # weakref to the owning WaterNet (not a registered child)
        object.__setattr__(self, "_slot", 0)

    def convs(self):
        return [getattr(self, f"conv{i}") for i in range(1, len(self.spec) + 1)]

    def _own_params(self):
        return [t for conv in self.convs() for t in (conv.weight, conv.bias)]

    def _bind(self, parent, slot: int) -> None:
        object.__setattr__(self, "_parent_ref", weakref.ref(parent))
        object.__setattr__(self, "_slot", slot)

    def __getstate__(self):  # pickling (torch.save(model)): the weakref to the parent is re-created by WaterNet
        state = self.__dict__.copy()
        state["_parent_ref"] = None
        return state

    def __deepcopy__(self, memo):  # a copy is free-standing until a WaterNet re-binds it (weakrefs do not deep-copy)
        ref, self.__dict__["_parent_ref"] = self.__dict__.get("_parent_ref"), None
        try:
            cls = type(self)
            new = cls.__new__(cls)
            memo[id(self)] = new
            import copy as _copy
            new.__dict__.update({k: _copy.deepcopy(v, memo) for k, v in self.__dict__.items()})
            return new
        finally:
            self.__dict__["_parent_ref"] = ref

    def _mode_and_engine(self, x, zero_layout):
        """(mode, engine with the right state dict packed, slot, tile or None).  zero_layout(own) -> the 34-tensor
        list of a free-standing stack."""
        parent = self._parent_ref() if self._parent_ref is not None else None
        if parent is not None:
            mode = parent._mode()
            return mode, parent._engine_with_weights(x), self._slot, _checked_tile(parent.tile, mode)
        if self.precision not in MODES:
            raise ValueError(f"unknown precision {self.precision!r}; choose from {sorted(MODES)}")
        mode = MODES[self.precision]
        tile = _checked_tile(self.tile, mode)
        own = self._own_params()
        return mode, self._engine_for(x, zero_layout(own), key_params=own), 0, tile

    def _train_engine(self, x, any_size=False):
        """(engine with the right state dict packed, slot) for a call that records an autograd graph, or None where
        the torch graph runs instead: CPU tensors, precision "fp32", or one image over Engine.TRAIN_MAX_PIXELS (unless
        ``any_size``: the windowed path)."""
        if not x.is_cuda or (not any_size and x.shape[2] * x.shape[3] > Engine.TRAIN_MAX_PIXELS):
            return None
        parent = self._parent_ref() if self._parent_ref is not None else None
        if parent is not None:
            if parent._mode() == _lib.MODE_FP32_SIMT:
                return None
            return parent._engine_with_weights(x), self._slot
        if self.precision not in MODES:
            raise ValueError(f"unknown precision {self.precision!r}; choose from {sorted(MODES)}")
        if MODES[self.precision] == _lib.MODE_FP32_SIMT:
            return None
        own = self._own_params()
        return self._engine_for(x, self._zero_layout(own), key_params=own), 0

    def _grad_tile(self):
        """The windowed-backward tile of a call that records an autograd graph, as (h, w), or None: the parent's
        ``grad_tile`` for a bound stack, else its own.  Refused with precision "fp32"."""
        parent = self._parent_ref() if self._parent_ref is not None else None
        if parent is not None:
            return _checked_grad_tile(parent.grad_tile, parent._mode())
        if self.precision not in MODES:
            raise ValueError(f"unknown precision {self.precision!r}; choose from {sorted(MODES)}")
        return _checked_grad_tile(self.grad_tile, MODES[self.precision])

    def _train_mode(self) -> int:
        """The training arithmetic (wn_set_train_mode) of a call that records an autograd graph: the parent's
        ``train_precision`` for a bound stack, else its own."""
        parent = self._parent_ref() if self._parent_ref is not None else None
        return parent._train_mode() if parent is not None else _checked_train_mode(self.train_precision)

    def _train_call(self, x):
        """(engine with the right state dict packed, slot, grad_tile or None, training mode) for a call that records
        an autograd graph, or None where the torch graph runs instead.  With grad_tile any image size runs natively."""
        grad_tile = self._grad_tile()
        native = self._train_engine(x, any_size=grad_tile is not None)
        return None if native is None else (*native, grad_tile, self._train_mode())

    @staticmethod
    def _needs_graph(tensors, params):
        return torch.is_grad_enabled() and (any(t.requires_grad for t in tensors) or any(p.requires_grad for p in params))


class _SubmoduleForward(torch.autograd.Function):
    """A sub-module called on its own under autograd: forward values and gradients from the CUDA library
    (wn_confidence_maps_train / _backward for the cmg, wn_refine_train / _backward for a refiner), in the bf16x3
    arithmetic of training.  It receives the stack's own 16 or 6 parameters, so autograd routes gradients to them and
    to nothing else.  which: None for the cmg, else the refiner slot (0 wb, 1 ce, 2 gc) of the packed state dict.
    With ``grad_tile`` the forward keeps nothing but the inputs (wn_confidence_maps_tiled / wn_refine_tiled in the
    bf16x3 arithmetic of training) and the backward recomputes the stack's activations window by window
    (wn_confidence_maps_backward_tiled / wn_refine_backward_tiled); both hold at most one pass of TRAIN_PASS_PIXELS
    window pixels.  train_mode (wn_set_train_mode) is kept for the backward, so that it runs under the forward's mode
    whatever another module trains on the same engine in between."""

    @staticmethod
    def forward(ctx, eng, which, grad_tile, train_mode, n_in, *tensors):
        ins, params = tensors[:n_in], tensors[n_in:]
        ctx.engine, ctx.which, ctx.n_in, ctx.grad_tile, ctx.train_mode = eng, which, n_in, grad_tile, train_mode
        ctx.weights_key = eng._weights_key
        ctx.shapes = [p.shape for p in params]
        if grad_tile is not None:
            ctx.save_for_backward(*ins)
            if which is None:
                return eng.confidence_maps_tiled(*ins, grad_tile, _lib.MODE_BF16X3, max_pass_pixels=TRAIN_PASS_PIXELS)
            return eng.refine_tiled(which, *ins, grad_tile, _lib.MODE_BF16X3, max_pass_pixels=TRAIN_PASS_PIXELS)
        if which is None:
            out, ctx.saved_ws = eng.confidence_maps_train(*ins, train_mode=train_mode)
        else:
            out, ctx.saved_ws = eng.refine_train(which, *ins, train_mode=train_mode)
        return out

    @staticmethod
    def backward(ctx, grad):
        eng = ctx.engine
        if eng._weights_key != ctx.weights_key:
            raise RuntimeError("sub-module parameters were modified between forward and backward")
        need = ctx.needs_input_grad[5:]
        want_in, want_par = need[:ctx.n_in], need[ctx.n_in:]
        tm = ctx.train_mode
        if ctx.grad_tile is not None:
            ins = ctx.saved_tensors
            if ctx.which is None:
                grads, gin = eng.confidence_maps_backward_tiled(grad, ins, ctx.shapes, ctx.grad_tile, want_in,
                                                                max_pass_pixels=TRAIN_PASS_PIXELS, train_mode=tm)
            else:
                grads, gin = eng.refine_backward_tiled(ctx.which, grad, ins, ctx.shapes, ctx.grad_tile, want_in,
                                                       max_pass_pixels=TRAIN_PASS_PIXELS, train_mode=tm)
        elif ctx.which is None:
            grads, gin = eng.confidence_maps_backward(grad, ctx.saved_ws, ctx.shapes, want_in, train_mode=tm)
        else:
            grads, gin = eng.refine_backward(ctx.which, grad, ctx.saved_ws, ctx.shapes, want_in, train_mode=tm)
        ctx.saved_ws = None
        return (None, None, None, None, None, *gin, *[g if w else None for g, w in zip(grads, want_par)])


def _zeros_like_spec(spec, ref):
    out = []
    for cin, cout, k in spec:
        out += [torch.zeros((cout, cin, k, k), dtype=torch.float32, device=ref.device),
                torch.zeros((cout,), dtype=torch.float32, device=ref.device)]
    return out


class ConfidenceMapGenerator(_ConvStack):
    """Eight convs, ReLU after the first seven, sigmoid after the last (net.py:7-56)."""

    spec = CMG_SPEC

    def _graph(self, x, wb, ce, gc):
        out = torch.cat([x, wb, ce, gc], dim=1)
        layers = self.convs()
        for conv in layers[:-1]:
            out = F.relu(conv(out))
        return torch.sigmoid(layers[-1](out))

    @staticmethod
    def _zero_layout(own):
        return own + 3 * _zeros_like_spec(REFINER_SPEC, own[0])

    def forward(self, x, wb, ce, gc):
        """Returns the three (N,1,H,W) maps ``out1, out2, out3`` like ``net.py:55-56``."""
        if self._needs_graph((x, wb, ce, gc), self._own_params()):
            native = self._train_call(x)
            if native is None:
                maps = self._graph(x, wb, ce, gc)
            else:
                eng, _, grad_tile, train_mode = native
                maps = _SubmoduleForward.apply(eng, None, grad_tile, train_mode, 4, x, wb, ce, gc, *self._own_params())
        else:
            mode, eng, _, tile = self._mode_and_engine(x, self._zero_layout)
            if tile is None:
                maps = eng.confidence_maps(x, wb, ce, gc, mode)
            else:
                maps = eng.confidence_maps_tiled(x, wb, ce, gc, tile, mode)
        return torch.split(maps, [1, 1, 1], dim=1)


class Refiner(_ConvStack):
    """Three conv+ReLU on cat[x, x_bar] (net.py:59-80); the last ReLU is part of it."""

    spec = REFINER_SPEC

    def _graph(self, x, xbar):
        out = torch.cat([x, xbar], dim=1)
        for conv in self.convs():
            out = F.relu(conv(out))
        return out

    @staticmethod
    def _zero_layout(own):  # a free-standing refiner runs in slot 0 (wb_refiner)
        return _zeros_like_spec(CMG_SPEC, own[0]) + own + 2 * _zeros_like_spec(REFINER_SPEC, own[0])

    def forward(self, x, xbar):
        if self._needs_graph((x, xbar), self._own_params()):
            native = self._train_call(x)
            if native is None:
                return self._graph(x, xbar)
            eng, slot, grad_tile, train_mode = native
            return _SubmoduleForward.apply(eng, slot, grad_tile, train_mode, 2, x, xbar, *self._own_params())
        mode, eng, slot, tile = self._mode_and_engine(x, self._zero_layout)
        if tile is None:
            return eng.refine(slot, x, xbar, mode)
        return eng.refine_tiled(slot, x, xbar, tile, mode)


class _KernelForward(torch.autograd.Function):
    """Forward values and all gradients (34 parameters, and the four input images when they require
    grad) from the CUDA library (wn_forward_train / wn_backward).  Only the fp32 CUDA-core mode obtains
    its gradients by re-evaluating the torch graph.  With ``grad_tile`` the forward keeps nothing but the four
    inputs (wn_forward_tiled in the bf16x3 arithmetic of training) and the backward recomputes the activations
    window by window (wn_backward_tiled); both hold at most one pass of TRAIN_PASS_PIXELS window pixels.  The native
    calls run in the model's ``train_precision``, kept in ctx for the backward.
    """

    @staticmethod
    def forward(ctx, model, mode, grad_tile, x, wb, ce, gc, *params):
        ctx.model = model
        ctx.native = mode != _lib.MODE_FP32_SIMT
        ctx.grad_tile = grad_tile
        ctx.train_mode = model._train_mode() if ctx.native else None
        ctx.input_needs_grad = [t.requires_grad for t in (x, wb, ce, gc)]
        if grad_tile is not None:
            eng = model._engine_with_weights(x)
            ctx.engine, ctx.weights_key = eng, eng._weights_key
            ctx.save_for_backward(x, wb, ce, gc)
            return eng.forward_tiled(x, wb, ce, gc, grad_tile, _lib.MODE_BF16X3, max_pass_pixels=TRAIN_PASS_PIXELS)
        if ctx.native:
            eng = model._engine_with_weights(x)
            out, ws = eng.forward_train(x, wb, ce, gc, train_mode=ctx.train_mode)
            ctx.engine, ctx.saved_ws = eng, ws
            ctx.weights_key = eng._weights_key
            return out
        ctx.save_for_backward(x, wb, ce, gc)
        return model._kernel_forward(x, wb, ce, gc, mode)

    @staticmethod
    def backward(ctx, grad_out):
        model = ctx.model
        params = list(model.parameters())
        if ctx.native:
            eng = ctx.engine
            if eng._weights_key != ctx.weights_key:  # parameters changed between forward and backward
                raise RuntimeError("model parameters were modified between forward and backward")
            want_in = any(ctx.input_needs_grad)
            shapes = [p.shape for p in params]
            if ctx.grad_tile is not None:
                res = eng.backward_tiled(grad_out, ctx.saved_tensors, shapes, ctx.grad_tile, want_input_grads=want_in,
                                         max_pass_pixels=TRAIN_PASS_PIXELS, train_mode=ctx.train_mode)
            else:
                res = eng.backward(grad_out, ctx.saved_ws, shapes, want_input_grads=want_in, train_mode=ctx.train_mode)
                ctx.saved_ws = None
            grads, gin = res if want_in else (res, [None] * 4)
            gpar = [g if p.requires_grad else None for g, p in zip(grads, params)]
            gin = [g if need else None for g, need in zip(gin, ctx.input_needs_grad)]
            return (None, None, None, *gin, *gpar)
        x, wb, ce, gc = ctx.saved_tensors
        with torch.enable_grad():
            ins = [t.detach().requires_grad_(t.requires_grad) for t in (x, wb, ce, gc)]
            out = model._graph(*ins)
            wanted = [t for t in ins if t.requires_grad] + [p for p in params if p.requires_grad]
            grads = torch.autograd.grad(out, wanted, grad_out, allow_unused=True)
        it = iter(grads)
        gin = [next(it) if t.requires_grad else None for t in ins]
        gpar = [next(it) if p.requires_grad else None for p in params]
        return (None, None, None, *gin, *gpar)


class _RaggedKernelForward(torch.autograd.Function):
    """``WaterNet.forward_many`` under autograd: the images of their own sizes through the ragged training step
    (wn_forward_train_ragged / wn_backward_ragged, the bf16x3 arithmetic of training).  Receives the four inputs of
    every item, flattened, then the 34 parameters; returns one output per item.  With ``grad_tile`` the forward keeps
    nothing but the inputs (wn_forward_ragged in the bf16x3 arithmetic of training) and the backward recomputes the
    activations window by window (wn_backward_ragged_tiled); both hold at most one pass of TRAIN_PASS_PIXELS slot
    pixels."""

    @staticmethod
    def forward(ctx, model, grad_tile, n_items, *tensors):
        flat, params = tensors[:4 * n_items], tensors[4 * n_items:]
        items = [flat[4 * i:4 * i + 4] for i in range(n_items)]
        eng = model._engine_with_weights(items[0][0])
        ctx.engine, ctx.weights_key, ctx.n_items, ctx.grad_tile = eng, eng._weights_key, n_items, grad_tile
        ctx.train_mode = model._train_mode()
        ctx.shapes = [p.shape for p in params]
        if grad_tile is not None:
            # refuse here what the backward would refuse (a window over the pixels of one training pass)
            sizes = [tuple(x.shape[2:]) for x, *_ in items for _ in range(x.shape[0]) if x.shape[2] * x.shape[3]]
            if sizes and eng.backward_ragged_tiled_workspace_bytes(sizes, grad_tile, TRAIN_PASS_PIXELS) == 0:
                raise _lib.WaterNetLibraryError(
                    f"forward_many: wn_backward_ragged_tiled rejects these images at grad_tile={grad_tile} (a window "
                    f"may have at most {Engine.TRAIN_MAX_PIXELS >> 20} Mi pixels); use a smaller grad_tile")
            ctx.save_for_backward(*flat)
            return tuple(eng.forward_ragged(items, grad_tile, _lib.MODE_BF16X3, max_pass_pixels=TRAIN_PASS_PIXELS))
        outs, ctx.saved_calls = eng.forward_train_ragged(items, train_mode=ctx.train_mode)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grad_outs):
        eng = ctx.engine
        if eng._weights_key != ctx.weights_key:  # parameters changed between forward and backward
            raise RuntimeError("model parameters were modified between forward and backward")
        need = ctx.needs_input_grad[3:]
        want_in = [need[4 * i:4 * i + 4] for i in range(ctx.n_items)]
        if ctx.grad_tile is not None:
            flat = ctx.saved_tensors
            items = [flat[4 * i:4 * i + 4] for i in range(ctx.n_items)]
            grads, gin = eng.backward_ragged_tiled(grad_outs, items, ctx.shapes, ctx.grad_tile, want_in,
                                                   max_pass_pixels=TRAIN_PASS_PIXELS, train_mode=ctx.train_mode)
        else:
            grads, gin = eng.backward_ragged(grad_outs, ctx.saved_calls, ctx.shapes, want_in, train_mode=ctx.train_mode)
            ctx.saved_calls = None
        gpar = [g if w else None for g, w in zip(grads, need[4 * ctx.n_items:])]
        return (None, None, None, *[t for row in gin for t in row], *gpar)


class WaterNet(_PackedWeightsMixin, nn.Module):
    """
    Gated fusion network (reference ``net.py:83-108``)::

        model = WaterNet().cuda()
        out = model(x, wb, he, gc)      # four (N,3,H,W) tensors -> (N,3,H,W)

    ``precision``: ``"default"`` = ``"bf16_fp8"`` (tensor cores: bf16 products of the operands' high parts,
    the two correction terms of the heavy layers as one fp8 MMA; ~4e-4 of the fp32 result, inside the 1e-3
    parity bar), ``"bf16x3"`` (all three terms in bf16, ~3e-5; what training always uses),
    ``"fp32"`` (CUDA-core fp32 FMA).

    ``tile``: None (whole images per pass, ~1.9 KB of workspace per pixel) or the largest output tile, an int or
    (h, w), e.g. 998.  When set, inference calls of the model and of its ``cmg`` and refiners run in overlapping
    windows (``wn_forward_tiled``): the same bits as untiled, with a workspace that does not grow with the image
    size (~15 GB at tile 998 for a 45 MP photo, which does not fit on an 80 GB card untiled).  Tensor-core
    precisions only.  A call that records an autograd graph (training) ignores ``tile`` and runs as without it.

    ``grad_tile``: None (a call that records an autograd graph keeps every activation until backward, ~5.6 KB per
    pixel, at most 8 Mi pixels per image) or the largest output tile of the windowed backward, an int or (h, w), e.g.
    998.  When set, such a call keeps only its four inputs; its output is ``wn_forward_tiled`` in the bf16x3
    arithmetic of training, and backward recomputes the activations window by window (``wn_backward_tiled``), in
    about 12 GB whatever the image or batch size.  The gradients equal the untiled ones up to the order of fp32 sums.
    It costs one more forward and the windows' overlap, so where the untiled path fits it is faster.  Tensor-core
    precisions only.  Calls of ``cmg`` and the refiners on their own follow it as well (``_ConvStack``).

    ``train_precision``: the arithmetic of the native training calls (forward, data gradients and weight gradients of
    every call that records an autograd graph, windowed and ragged ones included).  ``"bf16x3"`` (default, ~1e-5 of
    fp32) or ``"bf16"``: one bf16 tensor-core product per product with fp32 accumulation, the operands rounded to bf16
    once, as autocast trains convolutions (DESIGN.md 4.13).  The forward of a ``grad_tile`` call stays bf16x3 (it is
    ``wn_forward_tiled``); ``precision`` and inference are unaffected.  ``cmg`` and the refiners follow it.
    """

    tile = None  # models pickled before the attribute existed
    grad_tile = None
    train_precision = "bf16x3"

    def __init__(self, precision: str = "default", tile=None, grad_tile=None, train_precision: str = "bf16x3"):
        super().__init__()
        _checked_train_mode(train_precision)
        self.cmg = ConfidenceMapGenerator()
        self.wb_refiner = Refiner()
        self.ce_refiner = Refiner()
        self.gc_refiner = Refiner()
        self.precision = precision
        self.tile = tile
        self.grad_tile = grad_tile
        self.train_precision = train_precision
        if tile is not None:
            _checked_tile(tile, self._mode())
        if grad_tile is not None:
            _checked_grad_tile(grad_tile, self._mode())
        self._bind_children()

    def _bind_children(self) -> None:
        self.cmg._bind(self, 0)
        for slot, ref in enumerate((self.wb_refiner, self.ce_refiner, self.gc_refiner)):
            ref._bind(self, slot)

    def __deepcopy__(self, memo):
        cls = type(self)
        new = cls.__new__(cls)
        memo[id(self)] = new
        import copy as _copy
        new.__dict__.update({k: _copy.deepcopy(v, memo) for k, v in self.__dict__.items()})
        new._bind_children()
        return new

    # -- plumbing -----------------------------------------------------------------
    def _mode(self) -> int:
        if self.precision not in MODES:
            raise ValueError(f"unknown precision {self.precision!r}; choose from {sorted(MODES)}")
        return MODES[self.precision]

    def _train_mode(self) -> int:
        return _checked_train_mode(self.train_precision)

    def _ordered_params(self):
        """The 34 tensors in state-dict order (what wn_pack_weights expects)."""
        out = []
        for stack in (self.cmg, self.wb_refiner, self.ce_refiner, self.gc_refiner):
            for conv in stack.convs():
                out += [conv.weight, conv.bias]
        return out

    def _engine_with_weights(self, x):
        """This model's private engine on x's device, its current parameters packed (no-op when unchanged)."""
        return self._engine_for(x, self._ordered_params())

    def engine(self):
        """The private engine on the device the parameters live on, current parameters packed."""
        class _On:  # what _engine_for looks at
            pass
        on = _On()
        on.device = self.cmg.conv1.weight.device
        on.is_cuda = on.device.type == "cuda"
        if on.is_cuda and on.device.index is None:
            on.device = torch.device("cuda", torch.cuda.current_device())
        return self._engine_for(on, self._ordered_params())

    def __setstate__(self, state):
        super().__setstate__(state)
        self._bind_children()

    def _kernel_forward(self, x, wb, ce, gc, mode):
        return self._engine_with_weights(x).forward(x, wb, ce, gc, mode)

    def _graph(self, x, wb, ce, gc):
        """Differentiable torch-op evaluation, used only to obtain gradients."""
        cm = self.cmg._graph(x, wb, ce, gc)
        r_wb = self.wb_refiner._graph(x, wb)
        r_ce = self.ce_refiner._graph(x, ce)
        r_gc = self.gc_refiner._graph(x, gc)
        return r_wb * cm[:, 0:1] + r_ce * cm[:, 1:2] + r_gc * cm[:, 2:3]

    # -- reference signature: forward(x, wb, ce, gc), ce == histogram-equalised image ---
    def forward(self, x, wb, ce, gc):
        mode = self._mode()
        if x.numel() == 0 and x.is_cuda:  # empty batch: nothing to launch (torch's convs return empty too)
            return self._engine_with_weights(x).forward(x, wb, ce, gc, mode)
        needs_graph = torch.is_grad_enabled() and (
            any(t.requires_grad for t in (x, wb, ce, gc)) or any(p.requires_grad for p in self.parameters()))
        if needs_graph:  # tile does not apply: training keeps every activation of whole images, unless grad_tile
            grad_tile = _checked_grad_tile(self.grad_tile, mode)
            return _KernelForward.apply(self, mode, grad_tile, x, wb, ce, gc, *self.parameters())
        tile = _checked_tile(self.tile, mode)
        if tile is not None:
            return self._engine_with_weights(x).forward_tiled(x, wb, ce, gc, tile, mode)
        return self._kernel_forward(x, wb, ce, gc, mode)

    def forward_many(self, xs, wbs, ces, gcs) -> list:
        """``forward`` of images of their own sizes: four equally long lists of (N_i,3,H_i,W_i) tensors -> the list of
        the (N_i,3,H_i,W_i) outputs.  Without an autograd graph one ragged call runs them all (``wn_forward_ragged``,
        windows of ``tile``, or ``Engine.DEFAULT_TILE`` when that is None); each output equals ``model(...)`` of that
        item alone bit for bit.  With a graph the images go through the ragged training step in as few calls as fit
        ``Engine.TRAIN_MAX_PIXELS`` slot pixels each (``wn_forward_train_ragged`` / ``wn_backward_ragged``); gradients
        reach the parameters and the inputs that require grad, and the parameter gradients are the sum over the
        images.  Tensor-core precisions only.

        Cost under autograd: every training call keeps its whole activation workspace (~5.6 KB per slot pixel, slots
        padded up to 25 %) until backward, so the list holds the activations of all its images at once.  One ragged
        step pays off for small images, which leave SMs idle one at a time: on one H100 (700 W) 32 images of 64-160
        pixels per side took 0.84x the time of a per-image loop, while 32 of 64 x 64 to 512 x 384 took 1.12x and
        about 10x the peak memory (17.3 GB against 1.8).

        With ``grad_tile`` set such a call keeps only the inputs: the outputs are one ``wn_forward_ragged`` call in the
        bf16x3 arithmetic of training, and backward is one ``wn_backward_ragged_tiled`` call that recomputes the
        windows of all images, packed into passes of ``TRAIN_PASS_PIXELS`` slot pixels, in about 12 GB whatever the
        list.  Outputs and input gradients equal those of ``model(...)`` of each item under the same ``grad_tile``
        bit for bit; the parameter gradients are their sum up to the order of fp32 sums.  A list with a window over
        ``Engine.TRAIN_MAX_PIXELS`` is refused here, not in backward."""
        mode = self._mode()
        if mode == _lib.MODE_FP32_SIMT:
            raise ValueError("forward_many: ragged batches run on the tensor cores only, and precision='fp32' is the "
                             "CUDA-core mode; use precision='default' or 'bf16x3', or call the model per image")
        if not (len(xs) == len(wbs) == len(ces) == len(gcs)):
            raise ValueError("forward_many: xs, wbs, ces and gcs must have the same length")
        items = list(zip(xs, wbs, ces, gcs))
        if not items:
            return []
        x0 = items[0][0]
        if not x0.is_cuda:
            self._engine_for(x0, None)  # raises: there is no CPU path
        params = list(self.parameters())
        needs_graph = torch.is_grad_enabled() and (
            any(t.requires_grad for it in items for t in it) or any(p.requires_grad for p in params))
        if needs_graph:
            grad_tile = _checked_grad_tile(self.grad_tile, mode)
            return list(_RaggedKernelForward.apply(self, grad_tile, len(items), *[t for it in items for t in it],
                                                   *params))
        tile = _checked_tile(self.tile, mode) or Engine.DEFAULT_TILE
        return self._engine_with_weights(x0).forward_ragged(items, tile, mode)
