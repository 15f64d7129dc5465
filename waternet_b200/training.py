"""Training / scoring loops of the reference (train.py:26-152, score.py) on the CUDA forward.

The model's forward values and all of its gradients come from the CUDA library
(``wn_forward_train`` / ``wn_backward``: tensor-core forward that keeps its activations, data-gradient and
weight-gradient kernels; only ``precision="fp32"`` re-evaluates the torch graph for its backward).  The
VGG19 perceptual model, Adam and the metrics stay PyTorch: they are not on the
north-star path.
"""
from __future__ import annotations

import json
import warnings
from pathlib import Path
from typing import Dict

import numpy as np
import torch
import torch.nn as nn

from .metrics import psnr, ssim

TRAIN_METRICS_NAMES = ["mse", "ssim", "psnr", "perceptual_loss", "loss"]
VAL_METRICS_NAMES = ["mse", "ssim", "psnr", "perceptual_loss"]
_MEAN = (0.485, 0.456, 0.406)
_STD = (0.229, 0.224, 0.225)


def next_run_dir(root: Path) -> Path:
    """``root/<n>`` with n = 1 + the largest all-digit subdirectory (train.py:209-221)."""
    root.mkdir(exist_ok=True)
    taken = [int(p.name) for p in root.iterdir() if p.is_dir() and p.name.isdecimal()]
    return root / str(max(taken) + 1 if taken else 0)


class PerceptualModel(nn.Module):
    """VGG19 ``features`` without the final max-pool (train.py:254-263)."""

    def __init__(self, pretrained: bool = True):
        super().__init__()
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


def _normalize(x):
    mean = torch.tensor(_MEAN, device=x.device, dtype=x.dtype).view(1, 3, 1, 1)
    std = torch.tensor(_STD, device=x.device, dtype=x.dtype).view(1, 3, 1, 1)
    return (x - mean) / std


def perceptual_loss(vgg, out, ref):
    """mean((255 * (vgg(norm(out)) - vgg(norm(ref))))^2)  (train.py:110-122)."""
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


def batch_quality(out, ref):
    """(SSIM, PSNR) of a batch.  For lists of images: the mean of the per-image SSIMs, and the PSNR of the MSE
    pooled over every pixel of every image."""
    if not isinstance(out, list):
        return ssim(out, ref), psnr(out, ref, 1.0)
    s = torch.stack([ssim(o, r) for o, r in zip(out, ref)]).mean()
    sq = sum(torch.sum((o - r) ** 2) for o, r in zip(out, ref))
    mse = sq / sum(o.numel() for o in out)
    return s, 10.0 * torch.log10(1.0 / mse)


def train_one_epoch(model, loader, optimizer, scheduler, vgg, device, log=None) -> Dict[str, float]:
    """One epoch; a batch is five tensors, or five lists of images of their own sizes (GpuBatchLoader(ragged=True))."""
    model.train()
    totals = {k: 0.0 for k in TRAIN_METRICS_NAMES}
    for idx, batch in enumerate(loader):
        raw, wb, he, gc, ref = _to_device(batch, device)
        out = _forward(model, raw, wb, he, gc)
        loss, perc, mse = batch_losses(vgg, out, ref)
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        scheduler.step()  # per minibatch, like the reference (train.py:133)
        with torch.no_grad():
            s, p = batch_quality(out, ref)
            totals["loss"] += loss.item()
            totals["perceptual_loss"] += perc.item()
            totals["mse"] += mse.item()
            totals["ssim"] += s.item()
            totals["psnr"] += p.item()
        if log is not None and idx and idx % 10 == 0:
            log(f"  batch {idx}/{len(loader)} loss {loss.item():.4g}")
    return {k: v / max(len(loader), 1) for k, v in totals.items()}


def eval_one_epoch(model, loader, vgg, device) -> Dict[str, float]:
    """Validation pass; the perceptual loss is averaged over batches (the reference logs only the
    last batch divided by the batch count, train.py:71-74)."""
    model.eval()
    totals = {k: 0.0 for k in VAL_METRICS_NAMES}
    with torch.no_grad():
        for batch in loader:
            raw, wb, he, gc, ref = _to_device(batch, device)
            out = _forward(model, raw, wb, he, gc)
            _, perc, mse = batch_losses(vgg, out, ref)
            s, p = batch_quality(out, ref)
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
