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
from typing import List, NamedTuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .engine import AUTO_TILE, TRAIN_PASS_PIXELS, Engine, is_auto, new_engine

MODES = {"default": _lib.MODE_DEFAULT, "fp32": _lib.MODE_FP32_SIMT, "bf16x3": _lib.MODE_BF16X3,
         "bf16_fp8": _lib.MODE_BF16_FP8}
# the arithmetic of the native training calls (wn_set_train_mode): three bf16 products per product (~1e-5 of fp32),
# or one (operands rounded to bf16 once, fp32 accumulation, as autocast trains convolutions)
TRAIN_PRECISIONS = {"bf16x3": _lib.MODE_BF16X3, "bf16": _lib.MODE_BF16}


# model -> {device index: Engine}.  Every module that can be called on its own (WaterNet and, like in the
# reference, its sub-modules) has a private engine per device = its own packed-weight slot in the library.
# Kept outside the module so that copy.deepcopy / pickling of a model never touches a C handle.
_model_engines = weakref.WeakKeyDictionary()
_model_engines_lock = threading.Lock()


def _checked_tile(name: str, runs: str, tile, mode: int, auto=None):
    """``tile`` (the attribute ``name``) as (h, w), or None.  ``runs`` (the tiled forward, the windowed backward) runs
    on the tensor cores only.  "auto" gives ``auto()``, the choice of ``Engine.auto_tile`` for one call, or "auto"
    itself without ``auto`` (the setting checked outside a call)."""
    if tile is None:
        return None
    if is_auto(tile, name):
        return tile if auto is None else auto()
    if mode == _lib.MODE_FP32_SIMT:
        raise ValueError(f"{name}: {runs} runs on the tensor cores only, and precision='fp32' is the CUDA-core mode; "
                         f"use precision='default' or 'bf16x3', or {name}=None")
    return Engine._tile_hw(tile)


def _param_version(p) -> int:
    try:
        return p._version
    except RuntimeError:  # tensors created under torch.inference_mode() do not track versions
        return -1


def _needs_graph(tensors, params) -> bool:
    """Whether a call records an autograd graph: grad mode is on and an input or a parameter requires grad."""
    return torch.is_grad_enabled() and (any(t.requires_grad for t in tensors) or any(p.requires_grad for p in params))


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

    def _device_engine(self, device) -> Engine:
        """This module's private engine on the CUDA ``device``, created on first use."""
        with _model_engines_lock:
            per_dev = _model_engines.setdefault(self, {})
            eng = per_dev.get(device.index)
            if eng is None:
                eng = per_dev[device.index] = new_engine(device)
        return eng

    def _pack_key(self, params) -> tuple:
        """The packed-weight cache key of ``params``: the epoch, then data_ptr and _version of every tensor."""
        return (getattr(self, "_pack_epoch", 0),) + tuple((p.data_ptr(), _param_version(p)) for p in params)

    def _engine_for(self, device, params, key_params=None):
        """This module's private engine on ``device`` (that of the inputs) with ``params`` (34 tensors, state-dict
        order) packed.  The cache key is taken over ``key_params`` when given (a free-standing stack: its own
        parameters, not the zeros that fill the other slots)."""
        if device.type != "cuda":
            raise _lib.WaterNetLibraryError(
                f"{type(self).__name__}.forward got CPU tensors: waternet_b200 has no CPU path; move the model and "
                "inputs to a CUDA device (H100)")
        if params[0].device != device:
            raise RuntimeError(f"model parameters on {params[0].device}, inputs on {device}")
        eng = self._device_engine(device)
        eng.pack_weights(params, key=self._pack_key(params if key_params is None else key_params))
        return eng


class _NetModule(_PackedWeightsMixin, nn.Module):
    """What ``WaterNet`` and its stacks share: the settings of a call, each validated where it is read, from the
    module's owner (``_owner``: a stack bound to a ``WaterNet`` follows the parent's settings)."""

    def _owner(self):
        return self

    def _mode(self) -> int:
        precision = self._owner().precision
        if precision not in MODES:
            raise ValueError(f"unknown precision {precision!r}; choose from {sorted(MODES)}")
        return MODES[precision]

    def _train_mode(self) -> int:
        """The training arithmetic (wn_set_train_mode) of a call that records an autograd graph."""
        train_precision = self._owner().train_precision
        if train_precision not in TRAIN_PRECISIONS:
            raise ValueError(f"unknown train_precision {train_precision!r}; choose from {sorted(TRAIN_PRECISIONS)}")
        return TRAIN_PRECISIONS[train_precision]

    _auto_kind = "net"  # the kind of Engine.auto_tile for this module's calls

    def _auto(self, x, train: bool, sizes=None):
        """The resolver of "auto" for a call on ``x`` (its first input; None: no call) that records an autograd graph
        when ``train``: Engine.auto_tile of this module's kind on x's (n, h, w), or of forward_many's training calls on
        the images of ``sizes``.  None (whole images) for CPU tensors, which have no windowed path."""
        if x is None:
            return None
        mode = self._mode()

        def resolve():
            if not x.is_cuda or x.dim() != 4:
                return None
            train_mode = self._train_mode() if train else None
            kind, shapes = ("ragged", sizes) if sizes is not None else (self._auto_kind, (x.shape[0],) + x.shape[2:])
            return Engine.auto_tile(kind, shapes, mode, train_mode, device=x.device)
        return resolve

    def _tile(self, x=None):
        """The window tile of a call without an autograd graph on ``x`` (its first input), as (h, w), or None; "auto"
        is resolved from x's shape (and left as "auto" without x).  Refused with precision "fp32", except "auto"."""
        return _checked_tile("tile", "the tiled forward", self._owner().tile, self._mode(), self._auto(x, False))

    def _grad_tile(self, x=None, sizes=None):
        """The windowed-backward tile of a call that records an autograd graph, as ``_tile``; ``sizes``: the images of
        a forward_many call, [(h, w), ...].  Refused with precision "fp32", except "auto"."""
        return _checked_tile("grad_tile", "the windowed backward", self._owner().grad_tile, self._mode(),
                             self._auto(x, True, sizes))


class _Training(NamedTuple):
    """How one kind of call trains on the library: the ``Engine`` methods of its training forward, backward, windowed
    forward and windowed backward; the arguments before the tensors (a refiner's ``which``); and how its flat inputs
    map onto those methods."""
    train: str
    backward: str
    tiled: str
    backward_tiled: str
    lead: tuple = ()
    items: bool = False    # the inputs are items of four tensors, one output per item (forward_many)
    ask_all: bool = False  # the library is asked for all input gradients when any is needed (wn_backward*)
    owner: str = "model"   # whose parameters a changed weights key reports

    def group(self, flat):
        """The inputs (or their needs) of a call as its methods take them: a list of items of four, or a tuple."""
        return [flat[i:i + 4] for i in range(0, len(flat), 4)] if self.items else tuple(flat)


_NET_TRAINING = _Training("forward_train", "backward", "forward_tiled", "backward_tiled", ask_all=True)
_CMG_TRAINING = _Training("confidence_maps_train", "confidence_maps_backward", "confidence_maps_tiled",
                          "confidence_maps_backward_tiled", owner="sub-module")
_REFINER_TRAINING = tuple(_Training("refine_train", "refine_backward", "refine_tiled", "refine_backward_tiled",
                                    lead=(which,), owner="sub-module") for which in range(3))
_RAGGED_TRAINING = _Training("forward_train_ragged", "backward_ragged", "forward_ragged", "backward_ragged_tiled",
                             items=True)


class _NativeTraining(torch.autograd.Function):
    """A call that records an autograd graph, on the library's training calls of ``kind`` (a ``_Training``).  It
    receives the call's inputs, then the parameters it trains, so autograd routes gradients to them and to nothing
    else.  Without ``grad_tile`` the forward keeps its activations until backward (wn_forward_train,
    wn_confidence_maps_train, ...).  With ``grad_tile`` it keeps nothing but the inputs: the forward is the windowed
    forward in the bf16x3 arithmetic of training, and the backward recomputes the activations window by window; both
    hold at most one pass of TRAIN_PASS_PIXELS window pixels.  train_mode (wn_set_train_mode) is kept for the backward,
    so that it runs under the forward's mode whatever another module trains on the same engine in between."""

    @staticmethod
    def forward(ctx, kind, eng, grad_tile, train_mode, n_in, *tensors):
        ins, params = tensors[:n_in], tensors[n_in:]
        ctx.kind, ctx.engine, ctx.grad_tile, ctx.train_mode, ctx.n_in = kind, eng, grad_tile, train_mode, n_in
        ctx.weights_key = eng._weights_key
        ctx.shapes = [p.shape for p in params]
        args = (kind.group(ins),) if kind.items else ins
        if grad_tile is not None:
            ctx.save_for_backward(*ins)
            out = getattr(eng, kind.tiled)(*kind.lead, *args, grad_tile, _lib.MODE_BF16X3,
                                           max_pass_pixels=TRAIN_PASS_PIXELS)
        else:
            out, ctx.saved_ws = getattr(eng, kind.train)(*kind.lead, *args, train_mode=train_mode)
        return tuple(out) if kind.items else out

    @staticmethod
    def backward(ctx, *grad_outs):
        kind, eng = ctx.kind, ctx.engine
        if eng._weights_key != ctx.weights_key:
            raise RuntimeError(f"{kind.owner} parameters were modified between forward and backward")
        need_in, need_par = ctx.needs_input_grad[5:5 + ctx.n_in], ctx.needs_input_grad[5 + ctx.n_in:]
        grad = grad_outs if kind.items else grad_outs[0]
        want = any(need_in) if kind.ask_all else kind.group(need_in)
        if ctx.grad_tile is not None:
            res = getattr(eng, kind.backward_tiled)(*kind.lead, grad, kind.group(ctx.saved_tensors), ctx.shapes,
                                                    ctx.grad_tile, want, max_pass_pixels=TRAIN_PASS_PIXELS,
                                                    train_mode=ctx.train_mode)
        else:
            res = getattr(eng, kind.backward)(*kind.lead, grad, ctx.saved_ws, ctx.shapes, want,
                                              train_mode=ctx.train_mode)
            ctx.saved_ws = None
        grads, gin = (res, [None] * ctx.n_in) if kind.ask_all and not want else res
        if kind.items:
            gin = [t for row in gin for t in row]
        return (None,) * 5 + tuple(g if need else None for g, need in zip(gin, need_in)) + \
            tuple(g if need else None for g, need in zip(grads, need_par))


class _SubmoduleForward(_NativeTraining):
    """``_NativeTraining`` of a sub-module called on its own, under a name of its own in the autograd graph
    (``grad_fn``), so that a sub-module's native node can be told from the whole network's."""


# (in, out, kernel) of the confidence-map stack (reference net.py:12-42) and of a refiner (net.py:62-70)
CMG_SPEC = [(12, 128, 7), (128, 128, 5), (128, 128, 3), (128, 64, 1), (64, 64, 7), (64, 64, 5), (64, 64, 3), (64, 3, 3)]
REFINER_SPEC = [(6, 32, 7), (32, 32, 5), (32, 3, 3)]


def _same_conv(cin: int, cout: int, k: int) -> nn.Conv2d:
    return nn.Conv2d(cin, cout, kernel_size=k, stride=1, dilation=1, padding=k // 2)


class _ConvStack(_NetModule):
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
    ``grad_tile``; a free-standing one uses its own attributes.  "auto" chooses per call as ``WaterNet`` describes,
    from this stack's own workspace.
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

    def _owner(self):
        """The parent WaterNet of a bound stack, whose settings it follows, else the stack itself."""
        parent = self._parent_ref() if self._parent_ref is not None else None
        return self if parent is None else parent

    def _engine_and_slot(self, x):
        """(engine with the right state dict packed, slot) for a call on x: the parent's engine and this stack's slot
        for a bound stack, else its own engine with its parameters in slot 0 of its kind and zeros elsewhere."""
        owner = self._owner()
        if owner is not self:
            return owner._engine_with_weights(x), self._slot
        own = self._own_params()
        return self._engine_for(x.device, self._zero_layout(own), key_params=own), 0

    def _train_engine(self, x, any_size=False):
        """(engine with the right state dict packed, slot) for a call on x that records an autograd graph, or None
        where the torch graph runs instead: CPU tensors, precision "fp32", or one image over Engine.TRAIN_MAX_PIXELS
        (unless ``any_size``: the windowed path of ``grad_tile``)."""
        if (not x.is_cuda or (not any_size and x.shape[2] * x.shape[3] > Engine.TRAIN_MAX_PIXELS)
                or self._mode() == _lib.MODE_FP32_SIMT):
            return None
        return self._engine_and_slot(x)

    def _trained(self, ins):
        """The stack on ``ins`` recording an autograd graph: natively where ``_train_engine`` allows, else the torch
        graph."""
        grad_tile = self._grad_tile(ins[0])
        native = self._train_engine(ins[0], any_size=grad_tile is not None)
        if native is None:
            return self._graph(*ins)
        eng, slot = native
        return _SubmoduleForward.apply(self._training[slot], eng, grad_tile, self._train_mode(), len(ins), *ins,
                                       *self._own_params())


def _zeros_like_spec(spec, ref):
    out = []
    for cin, cout, k in spec:
        out += [torch.zeros((cout, cin, k, k), dtype=torch.float32, device=ref.device),
                torch.zeros((cout,), dtype=torch.float32, device=ref.device)]
    return out


class ConfidenceMapGenerator(_ConvStack):
    """Eight convs, ReLU after the first seven, sigmoid after the last (net.py:7-56)."""

    spec = CMG_SPEC
    _training = (_CMG_TRAINING,)
    _auto_kind = "cmg"

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
        ins = (x, wb, ce, gc)
        if _needs_graph(ins, self._own_params()):
            maps = self._trained(ins)
        else:
            mode, tile = self._mode(), self._tile(x)
            eng, _ = self._engine_and_slot(x)
            maps = eng.confidence_maps(*ins, mode) if tile is None else eng.confidence_maps_tiled(*ins, tile, mode)
        return torch.split(maps, [1, 1, 1], dim=1)


class Refiner(_ConvStack):
    """Three conv+ReLU on cat[x, x_bar] (net.py:59-80); the last ReLU is part of it."""

    spec = REFINER_SPEC
    _training = _REFINER_TRAINING  # by slot (0 wb, 1 ce, 2 gc)
    _auto_kind = "refiner"

    def _graph(self, x, xbar):
        out = torch.cat([x, xbar], dim=1)
        for conv in self.convs():
            out = F.relu(conv(out))
        return out

    @staticmethod
    def _zero_layout(own):  # a free-standing refiner runs in slot 0 (wb_refiner)
        return _zeros_like_spec(CMG_SPEC, own[0]) + own + 2 * _zeros_like_spec(REFINER_SPEC, own[0])

    def forward(self, x, xbar):
        if _needs_graph((x, xbar), self._own_params()):
            return self._trained((x, xbar))
        mode, tile = self._mode(), self._tile(x)
        eng, slot = self._engine_and_slot(x)
        return eng.refine(slot, x, xbar, mode) if tile is None else eng.refine_tiled(slot, x, xbar, tile, mode)


class _GraphBackward(torch.autograd.Function):
    """``WaterNet`` in precision "fp32" under autograd: the forward on the fp32 CUDA-core kernels, the gradients (34
    parameters and the inputs that require grad) by re-evaluating the torch graph (``model._graph``)."""

    @staticmethod
    def forward(ctx, model, x, wb, ce, gc, *params):
        ctx.model = model
        ctx.save_for_backward(x, wb, ce, gc)
        return model._engine_with_weights(x).forward(x, wb, ce, gc, _lib.MODE_FP32_SIMT)

    @staticmethod
    def backward(ctx, grad_out):
        params = list(ctx.model.parameters())
        with torch.enable_grad():
            ins = [t.detach().requires_grad_(t.requires_grad) for t in ctx.saved_tensors]
            out = ctx.model._graph(*ins)
            wanted = [t for t in ins if t.requires_grad] + [p for p in params if p.requires_grad]
            grads = torch.autograd.grad(out, wanted, grad_out, allow_unused=True)
        it = iter(grads)
        gin = [next(it) if t.requires_grad else None for t in ins]
        gpar = [next(it) if p.requires_grad else None for p in params]
        return (None, *gin, *gpar)


class WaterNet(_NetModule):
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

    ``tile="auto"`` / ``grad_tile="auto"`` choose per call, from the input's shape (``Engine.auto_tile``): whole images
    where the whole-image path's workspace for the call (for training: every activation it keeps) is at most
    ``Engine.AUTO_WORKSPACE_BYTES`` (None: half the card's memory), else windows of ``Engine.DEFAULT_TILE``; a call the
    whole-image path refuses (an image over 8 Mi pixels under autograd) takes windows.  With ``precision="fp32"``
    "auto" always means whole images.  ``forward_many`` decides ``grad_tile`` once for its whole list.

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
        self.precision = precision
        self.tile = tile
        self.grad_tile = grad_tile
        self.train_precision = train_precision
        self._train_mode()
        if tile is not None:
            self._tile()
        if grad_tile is not None:
            self._grad_tile()
        self.cmg = ConfidenceMapGenerator()
        self.wb_refiner = Refiner()
        self.ce_refiner = Refiner()
        self.gc_refiner = Refiner()
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
    def _ordered_params(self):
        """The 34 tensors in state-dict order (what wn_pack_weights expects)."""
        out = []
        for stack in (self.cmg, self.wb_refiner, self.ce_refiner, self.gc_refiner):
            for conv in stack.convs():
                out += [conv.weight, conv.bias]
        return out

    def _engine_with_weights(self, x):
        """This model's private engine on x's device, its current parameters packed (no-op when unchanged)."""
        return self._engine_for(x.device, self._ordered_params())

    def engine(self):
        """The private engine on the device the parameters live on, current parameters packed."""
        return self._engine_for(self.cmg.conv1.weight.device, self._ordered_params())

    def __setstate__(self, state):
        super().__setstate__(state)
        self._bind_children()

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
        ins = (x, wb, ce, gc)
        if x.numel() == 0 and x.is_cuda:  # empty batch: nothing to launch (torch's convs return empty too)
            return self._engine_with_weights(x).forward(*ins, mode)
        # tile does not apply to training: it keeps every activation of whole images, unless grad_tile
        if _needs_graph(ins, self.parameters()):
            grad_tile = self._grad_tile(x)
            if mode == _lib.MODE_FP32_SIMT:
                return _GraphBackward.apply(self, *ins, *self.parameters())
            train_mode = self._train_mode()
            return _NativeTraining.apply(_NET_TRAINING, self._engine_with_weights(x), grad_tile, train_mode, 4, *ins,
                                         *self.parameters())
        tile = self._tile(x)
        eng = self._engine_with_weights(x)
        return eng.forward(*ins, mode) if tile is None else eng.forward_tiled(*ins, tile, mode)

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
            self._engine_for(x0.device, None)  # raises: there is no CPU path
        flat = [t for it in items for t in it]
        if _needs_graph(flat, self.parameters()):
            sizes = [] if self.grad_tile is None else \
                [tuple(x.shape[2:]) for x, *_ in items for _ in range(x.shape[0]) if x.shape[2] * x.shape[3]]
            grad_tile = self._grad_tile(x0, sizes)  # "auto": once for the whole list, kept in ctx for backward
            eng = self._engine_with_weights(x0)
            train_mode = self._train_mode()
            if grad_tile is not None:  # refuse here what the backward would refuse (a window over one training pass)
                if sizes and eng.backward_ragged_tiled_workspace_bytes(sizes, grad_tile, TRAIN_PASS_PIXELS) == 0:
                    raise _lib.WaterNetLibraryError(
                        f"forward_many: wn_backward_ragged_tiled rejects these images at grad_tile={grad_tile} (a "
                        f"window may have at most {Engine.TRAIN_MAX_PIXELS >> 20} Mi pixels); use a smaller grad_tile")
            return list(_NativeTraining.apply(_RAGGED_TRAINING, eng, grad_tile, train_mode, len(flat), *flat,
                                              *self.parameters()))
        tile = self._tile()
        tile = Engine.DEFAULT_TILE if tile is None or tile == AUTO_TILE else tile
        return self._engine_with_weights(x0).forward_ragged(items, tile, mode)
