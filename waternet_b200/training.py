"""Training / scoring loops of the reference (train.py:26-152, score.py) on the CUDA forward.

The model's forward values and all of its gradients come from the CUDA library
(``wn_forward_train`` / ``wn_backward``: tensor-core forward that keeps its activations, data-gradient and
weight-gradient kernels; only ``precision="fp32"`` re-evaluates the torch graph for its backward).  The
VGG19 perceptual loss is the torch expression by default; ``PerceptualModel(native=True)`` computes it and its
gradient in overlapping windows on the library's kernels (``wn_perceptual_loss``).  SSIM and PSNR are the torch
expressions of ``metrics`` by default; ``native=True`` (``--metrics native``) computes them with ``wn_quality``.
``ssim_weight`` (``--ssim-weight``) adds ``ssim_weight * metrics.ssim_loss(out, ref)`` to the loss, 1 - SSIM and its
gradient from ``wn_ssim_grad``.  Adam stays PyTorch.
"""
from __future__ import annotations

import argparse
import json
import warnings
from pathlib import Path
from typing import Dict

import numpy as np
import torch
import torch.nn as nn

from .engine import AUTO_TILE, Engine, is_auto
from .metrics import native_quality, psnr, ssim, ssim_loss
from .net import TRAIN_PRECISIONS, _PackedWeightsMixin

TRAIN_METRICS_NAMES = ["mse", "ssim", "psnr", "perceptual_loss", "loss"]
VAL_METRICS_NAMES = ["mse", "ssim", "psnr", "perceptual_loss"]
_MEAN = (0.485, 0.456, 0.406)
_STD = (0.229, 0.224, 0.225)


def next_run_dir(root: Path) -> Path:
    """``root/<n>`` with n = 1 + the largest all-digit subdirectory (train.py:209-221)."""
    root.mkdir(exist_ok=True)
    taken = [int(p.name) for p in root.iterdir() if p.is_dir() and p.name.isdecimal()]
    return root / str(max(taken) + 1 if taken else 0)


class PerceptualModel(_PackedWeightsMixin, nn.Module):
    """VGG19 ``features`` without the final max-pool (train.py:254-263).

    ``native=True``: on CUDA tensors ``perceptual_loss(vgg, out, ref)`` is one ``wn_perceptual_loss`` call -- the
    loss and d(loss)/d(out) on the tensor cores (``precision``), in windows that own ``tile`` input pixels of features
    (None: one window per image; an image over 8 Mi pixels then needs a tile), so memory is bounded by one pass
    whatever the image and batch size.  Autograd keeps only d(out), 12 bytes per pixel; no VGG weight gradient is
    computed (the VGG parameters' ``.grad`` stays untouched) and ``ref`` is a constant.  ``native=False`` and CPU
    tensors evaluate the torch expression.  ``tile="auto"`` chooses per call (``Engine.auto_tile``): one window per
    image where that workspace fits ``Engine.AUTO_WORKSPACE_BYTES`` (None: half the card's memory) and the call is
    allowed, else windows of ``Engine.DEFAULT_TILE``.

    ``precision``: the arithmetic of the native calls' 32 VGG convolutions.  "bf16x3" (default) issues three bf16
    tensor-core products per product; "bf16" issues one, a_hi x w_hi with fp32 accumulation, as autocast runs a frozen
    VGG (DESIGN.md 4.14).  "bf16" needs ``native=True``: the torch expression has its own arithmetic.  Read at every
    call, so a change takes effect at the next one."""

    precision = "bf16x3"  # class default: a module pickled before the attribute existed loads as bf16x3

    def __init__(self, pretrained: bool = True, native: bool = False, tile=None, precision: str = "bf16x3"):
        super().__init__()
        self.native = native
        self.tile = tile
        self.precision = precision
        self._train_mode()
        is_auto(tile)  # a string other than "auto" is refused here
        import torchvision
        vgg = None
        if pretrained:
            try:
                vgg = torchvision.models.vgg19(weights=torchvision.models.VGG19_Weights.IMAGENET1K_V1)
            except Exception as exc:  # offline: no checkpoint can be fetched
                warnings.warn(f"VGG19 ImageNet weights unavailable ({exc}); using a seeded random init")
        if vgg is None:
            state = torch.random.get_rng_state()
            torch.manual_seed(1234)
            vgg = torchvision.models.vgg19(weights=None)
            torch.random.set_rng_state(state)
        self.model = nn.Sequential(*list(vgg.features.children())[:-1])

    def forward(self, x):
        return self.model(x)

    def _train_mode(self) -> int:
        """The wn_set_train_mode of ``precision`` for the native calls; ValueError for an unknown value or for "bf16"
        without ``native``."""
        if self.precision not in TRAIN_PRECISIONS:
            raise ValueError(f"unknown precision {self.precision!r}; choose from {sorted(TRAIN_PRECISIONS)}")
        if self.precision != "bf16x3" and not self.native:
            raise ValueError(f"precision={self.precision!r} needs native=True: the torch expression (native=False) "
                             "has its own arithmetic")
        return TRAIN_PRECISIONS[self.precision]

    def vgg_params(self):
        """Weight and bias of the 16 convolutions in ``features`` order."""
        return [t for m in self.model if isinstance(m, nn.Conv2d) for t in (m.weight, m.bias)]

    def _vgg_engine(self, x):
        """This module's engine on x's device with the VGG weights packed; re-packed when the cache key of
        ``_PackedWeightsMixin`` (epoch, data_ptr and _version of every parameter) changes."""
        params = self.vgg_params()
        if params[0].device != x.device:
            raise RuntimeError(f"VGG parameters on {params[0].device}, inputs on {x.device}")
        eng = self._device_engine(x.device)
        eng.pack_vgg_weights(params, key=self._pack_key(params))
        return eng

    def _loss_tile(self, out):
        """``tile`` of a native call on ``out``, with "auto" resolved for its shape."""
        if not is_auto(self.tile):
            return self.tile
        n, _, h, w = out.shape
        return Engine.auto_tile("vgg", (n, h, w), self._train_mode(), device=out.device)

    def native_loss(self, out, ref):
        """The loss of ``perceptual_loss`` from one ``wn_perceptual_loss`` call (autograd: d(out) only)."""
        want = torch.is_grad_enabled() and out.requires_grad
        return _NativePerceptualLoss.apply(out, ref, self, want)


class _NativePerceptualLoss(torch.autograd.Function):
    """forward: one wn_perceptual_loss call; keeps d(loss)/d(out) when out needs a gradient, nothing else.
    backward: grad_output * d(out)."""

    @staticmethod
    def forward(ctx, out, ref, vgg, want_grad):
        loss, grad = vgg._vgg_engine(out).perceptual_loss(out, ref, tile=vgg._loss_tile(out), want_grad=want_grad,
                                                          train_mode=vgg._train_mode())
        if grad is not None:
            ctx.save_for_backward(grad)
        return loss

    @staticmethod
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        return grad_output * grad, None, None, None


def tile_arg(text: str):
    """The argparse type of --tile, --grad-tile and --perceptual-tile: "auto", or an int (checked where it is used)."""
    if text == AUTO_TILE:
        return text
    try:
        return int(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected {AUTO_TILE!r} or an integer, got {text!r}") from None


def add_perceptual_args(ap) -> None:
    """``--perceptual {torch,native}``, ``--perceptual-tile N`` and ``--perceptual-precision {bf16x3,bf16}`` of train.py
    and score.py."""
    ap.add_argument("--perceptual", default="torch", choices=["torch", "native"],
                    help="(Optional) torch: the perceptual loss as the torch VGG19 expression (default); native: the "
                         "loss and its gradient on the library's kernels in overlapping windows "
                         "(PerceptualModel(native=True)), memory bounded by one pass")
    ap.add_argument("--perceptual-tile", type=tile_arg, default=None, metavar="N|auto",
                    help="(Optional) needs --perceptual native: windows owning N x N input pixels of VGG features "
                         "(rounded up to a multiple of 16).  auto: one window per image where that fits half the "
                         "card's memory, else N = 998, chosen per call.  Unset: one window per image")
    ap.add_argument("--perceptual-precision", default=None, choices=sorted(TRAIN_PRECISIONS),
                    help="(Optional) needs --perceptual native: the arithmetic of the VGG convolutions "
                         "(PerceptualModel.precision), bf16x3 (default, three bf16 tensor-core products per product) "
                         "or bf16 (one, fp32 accumulation).  --train-precision does not set it")


def perceptual_model(args) -> PerceptualModel:
    """The PerceptualModel the command-line arguments of ``add_perceptual_args`` ask for; --perceptual-tile and
    --perceptual-precision without --perceptual native are refused (the torch expression has no windows and its own
    arithmetic)."""
    if args.perceptual_tile is not None and args.perceptual != "native":
        raise SystemExit("--perceptual-tile needs --perceptual native")
    if args.perceptual_tile not in (None, AUTO_TILE) and args.perceptual_tile <= 0:
        raise SystemExit("--perceptual-tile must be positive")
    if args.perceptual_precision is not None and args.perceptual != "native":
        raise SystemExit("--perceptual-precision needs --perceptual native")
    return PerceptualModel(native=args.perceptual == "native", tile=args.perceptual_tile,
                           precision=perceptual_config(args)["perceptual_precision"])


def add_metrics_arg(ap) -> None:
    """``--metrics {torch,native}`` of train.py and score.py."""
    ap.add_argument("--metrics", default="torch", choices=["torch", "native"],
                    help="(Optional) torch: SSIM and PSNR as the torch expressions (default); native: one wn_quality "
                         "call per batch on the library's kernels, no per-pixel temporaries")


def metrics_config(args) -> dict:
    """The metric setting of ``add_metrics_arg`` as train.py records it in config.json."""
    return {"metrics": args.metrics}


def _nonnegative(text: str) -> float:
    try:
        v = float(text)
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected a number, got {text!r}") from None
    if not v >= 0 or v == float("inf"):
        raise argparse.ArgumentTypeError(f"must be finite and at least 0, got {text!r}")
    return v


def add_loss_arg(ap) -> None:
    """``--ssim-weight W`` of train.py."""
    ap.add_argument("--ssim-weight", type=_nonnegative, default=0.0, metavar="W",
                    help="(Optional) Add W * (1 - SSIM) to the loss, SSIM and its gradient on the library's kernels "
                         "(metrics.ssim_loss), no per-pixel temporaries besides d(out).  Default 0: the reference's "
                         "0.05 * perceptual + mse, nothing extra computed")


def loss_config(args) -> dict:
    """The loss setting of ``add_loss_arg`` as train.py records it in config.json."""
    return {"ssim_weight": args.ssim_weight}


def perceptual_config(args) -> dict:
    """The perceptual-loss settings of ``add_perceptual_args`` as train.py records them in config.json."""
    return {"perceptual": args.perceptual, "perceptual_tile": args.perceptual_tile,
            "perceptual_precision": args.perceptual_precision or "bf16x3"}


def _normalize(x):
    mean = torch.tensor(_MEAN, device=x.device, dtype=x.dtype).view(1, 3, 1, 1)
    std = torch.tensor(_STD, device=x.device, dtype=x.dtype).view(1, 3, 1, 1)
    return (x - mean) / std


def perceptual_loss(vgg, out, ref):
    """mean((255 * (vgg(norm(out)) - vgg(norm(ref))))^2)  (train.py:110-122).  A ``PerceptualModel(native=True)``
    takes CUDA tensors to ``wn_perceptual_loss`` instead."""
    if getattr(vgg, "native", False) and out.is_cuda:
        return vgg.native_loss(out, ref)
    return torch.mean(torch.square(255 * (vgg(_normalize(out)) - vgg(_normalize(ref)))))


def _to_device(batch, device):
    """The five batch entries on ``device``: tensors, or lists of per-image tensors (a ragged batch)."""
    def move(v):
        return [t.to(device, non_blocking=True) for t in v] if isinstance(v, (list, tuple)) else \
            v.to(device, non_blocking=True)
    return [move(batch[k]) for k in ("raw", "wb", "he", "gc", "ref")]


def _forward(model, raw, wb, he, gc):
    """model(...) of a tensor batch; WaterNet.forward_many of a ragged batch (lists of images)."""
    return model.forward_many(raw, wb, he, gc) if isinstance(raw, list) else model(raw, wb, he, gc)


def batch_losses(vgg, out, ref):
    """(loss, perceptual loss, mse) of a batch, train.py:110-125.  For lists of images (a ragged batch) each term is
    the mean over the images of that image's term, so loss = mean_i(0.05 perc_i + mse_i): the reference's batch loss
    when all images have one size."""
    if not isinstance(out, list):
        perc = perceptual_loss(vgg, out, ref)
        mse = torch.mean(torch.square(255 * (out - ref)))
        return 0.05 * perc + mse, perc, mse
    perc = torch.stack([perceptual_loss(vgg, o, r) for o, r in zip(out, ref)])
    mse = torch.stack([torch.mean(torch.square(255 * (o - r))) for o, r in zip(out, ref)])
    return (0.05 * perc + mse).mean(), perc.mean(), mse.mean()


def batch_quality(out, ref, native: bool = False):
    """(SSIM, PSNR) of a batch.  For lists of images: the mean of the per-image SSIMs, and the PSNR of the MSE
    pooled over every pixel of every image.  ``native``: both from one ``metrics.native_quality`` call (CUDA tensors
    only; float64 results)."""
    if native:
        return native_quality(out, ref)
    if not isinstance(out, list):
        return ssim(out, ref), psnr(out, ref, 1.0)
    s = torch.stack([ssim(o, r) for o, r in zip(out, ref)]).mean()
    sq = sum(torch.sum((o - r) ** 2) for o, r in zip(out, ref))
    mse = sq / sum(o.numel() for o in out)
    return s, 10.0 * torch.log10(1.0 / mse)


def train_one_epoch(model, loader, optimizer, scheduler, vgg, device, log=None,
                    native_metrics: bool = False, ssim_weight: float = 0.0) -> Dict[str, float]:
    """One epoch; a batch is five tensors, or five lists of images of their own sizes (GpuBatchLoader(ragged=True)).
    ``native_metrics``: SSIM and PSNR from ``batch_quality(native=True)``.  ``ssim_weight``: the loss is
    ``0.05 * perc + mse + ssim_weight * metrics.ssim_loss(out, ref)`` (1 - SSIM of ``batch_quality``'s semantics);
    at 0 nothing extra is computed."""
    model.train()
    totals = {k: 0.0 for k in TRAIN_METRICS_NAMES}
    for idx, batch in enumerate(loader):
        raw, wb, he, gc, ref = _to_device(batch, device)
        out = _forward(model, raw, wb, he, gc)
        loss, perc, mse = batch_losses(vgg, out, ref)
        if ssim_weight:
            loss = loss + ssim_weight * ssim_loss(out, ref)
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        scheduler.step()  # per minibatch, like the reference (train.py:133)
        with torch.no_grad():
            s, p = batch_quality(out, ref, native_metrics)
            totals["loss"] += loss.item()
            totals["perceptual_loss"] += perc.item()
            totals["mse"] += mse.item()
            totals["ssim"] += s.item()
            totals["psnr"] += p.item()
        if log is not None and idx and idx % 10 == 0:
            log(f"  batch {idx}/{len(loader)} loss {loss.item():.4g}")
    return {k: v / max(len(loader), 1) for k, v in totals.items()}


def eval_one_epoch(model, loader, vgg, device, native_metrics: bool = False) -> Dict[str, float]:
    """Validation pass; the perceptual loss is averaged over batches (the reference logs only the
    last batch divided by the batch count, train.py:71-74).  ``native_metrics`` as ``train_one_epoch``."""
    model.eval()
    totals = {k: 0.0 for k in VAL_METRICS_NAMES}
    with torch.no_grad():
        for batch in loader:
            raw, wb, he, gc, ref = _to_device(batch, device)
            out = _forward(model, raw, wb, he, gc)
            _, perc, mse = batch_losses(vgg, out, ref)
            s, p = batch_quality(out, ref, native_metrics)
            totals["perceptual_loss"] += perc.item()
            totals["mse"] += mse.item()
            totals["ssim"] += s.item()
            totals["psnr"] += p.item()
    model.train()
    return {k: v / max(len(loader), 1) for k, v in totals.items()}


def save_metrics(savedir: Path, train_hist, val_hist, config: dict) -> None:
    """metrics-train.csv, metrics-val.csv, config.json (train.py:311-348)."""
    savedir.mkdir(parents=True, exist_ok=True)
    for fname, names, hist in (("metrics-train.csv", TRAIN_METRICS_NAMES, train_hist),
                               ("metrics-val.csv", VAL_METRICS_NAMES, val_hist)):
        if hist is None:
            continue
        arr = np.array([[row[n] for n in names] for row in hist], dtype=np.float64).reshape(-1, len(names))
        np.savetxt(savedir / fname, arr, fmt="%f", delimiter=",", comments="", header=",".join(names))
    with open(savedir / "config.json", "w") as f:
        json.dump(config, f, indent=4)
