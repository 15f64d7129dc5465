"""SSIM / PSNR as the reference's training loop uses them (train.py:139-144), without torchmetrics.

``structural_similarity_index_measure(preds, target)`` defaults: 11x11 gaussian window,
sigma 1.5, k1 0.01, k2 0.03, data range inferred as max(preds.max()-preds.min(),
target.max()-target.min()), reflect padding cropped away, mean over the batch.
``peak_signal_noise_ratio(preds, target, data_range=1)``: 10*log10(1/mse) over all elements.

``native_quality`` computes the same two numbers on the library's kernels (``wn_quality``, DESIGN.md 4.16), and
``ssim_loss`` the training loss 1 - SSIM and its gradient (``wn_ssim_grad``, DESIGN.md 4.17).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _gaussian_window(size: int, sigma: float, channels: int, device, dtype):
    coords = torch.arange(size, device=device, dtype=dtype) - (size - 1) / 2
    g = torch.exp(-(coords ** 2) / (2 * sigma ** 2))
    g = g / g.sum()
    k = torch.outer(g, g)
    return k.expand(channels, 1, size, size).contiguous()


def ssim(preds: torch.Tensor, target: torch.Tensor, kernel_size: int = 11, sigma: float = 1.5,
         k1: float = 0.01, k2: float = 0.03) -> torch.Tensor:
    c = preds.shape[1]
    data_range = torch.maximum(preds.max() - preds.min(), target.max() - target.min())
    c1, c2 = (k1 * data_range) ** 2, (k2 * data_range) ** 2
    pad = (kernel_size - 1) // 2
    win = _gaussian_window(kernel_size, sigma, c, preds.device, preds.dtype)
    p = F.pad(preds, (pad, pad, pad, pad), mode="reflect")
    t = F.pad(target, (pad, pad, pad, pad), mode="reflect")
    stack = torch.cat([p, t, p * p, t * t, p * t])
    out = F.conv2d(stack, win, groups=c)
    n = preds.shape[0]
    mu_p, mu_t, e_pp, e_tt, e_pt = (out[i * n:(i + 1) * n] for i in range(5))
    var_p, var_t, cov = e_pp - mu_p ** 2, e_tt - mu_t ** 2, e_pt - mu_p * mu_t
    s = ((2 * mu_p * mu_t + c1) * (2 * cov + c2)) / ((mu_p ** 2 + mu_t ** 2 + c1) * (var_p + var_t + c2))
    s = s[..., pad:-pad, pad:-pad] if s.shape[-1] > 2 * pad and s.shape[-2] > 2 * pad else s
    return s.reshape(n, -1).mean(-1).mean()


def psnr(preds: torch.Tensor, target: torch.Tensor, data_range: float = 1.0) -> torch.Tensor:
    mse = torch.mean((preds - target) ** 2)
    return 10.0 * torch.log10(data_range ** 2 / mse)


def _check_pair(o, r, what: str) -> None:
    """ValueError unless ``o`` and ``r`` are (N,3,H,W) of one shape with both sides above 5 (the reflect padding of
    ``ssim`` refuses a side of 5 or less)."""
    if o.dim() != 4 or o.shape[1] != 3 or o.shape != r.shape:
        raise ValueError(f"{what}: expected out and ref of one (N,3,H,W) shape, got {tuple(o.shape)} and "
                         f"{tuple(r.shape)}")
    if o.shape[0] == 0:
        raise ValueError(f"{what}: empty batch")
    if min(o.shape[2:]) <= 5:
        raise ValueError(f"{what}: padding size should be less than the corresponding input dimension, but got "
                         f"padding (5, 5) for input {list(o.shape)}: both sides must be at least 6")


def _native_pairs(out, ref, what: str):
    """The engine and the flat per-image lists of a ``native_quality`` / ``ssim_loss`` call: (engine, items, outs,
    refs, groups, counts), with items the (out, ref) pairs as given, outs and refs detached fp32 contiguous (3,H,W)
    images, groups their item indices and counts the images per item."""
    from .engine import get_engine

    if isinstance(out, (list, tuple)):
        if not isinstance(ref, (list, tuple)) or len(out) != len(ref) or not out:
            raise ValueError(f"{what}: expected two equally long, non-empty lists of (N_i,3,H_i,W_i) tensors")
        items = list(zip(out, ref))
    else:
        items = [(out, ref)]
    for k, (o, r) in enumerate(items):
        _check_pair(o, r, f"{what} (item {k})" if len(items) > 1 else what)
    eng = get_engine(items[0][0].device)
    outs, refs, groups, counts = [], [], [], []
    for k, (o, r) in enumerate(items):
        if o.device != eng.device or r.device != eng.device:
            raise ValueError(f"{what}: every tensor must be on {eng.device}, item {k} is on {o.device} and "
                             f"{r.device}")
        o, r = (t.detach().to(torch.float32).contiguous() for t in (o, r))
        outs += list(o)
        refs += list(r)
        groups += [k] * o.shape[0]
        counts.append(o.shape[0])
    return eng, items, outs, refs, groups, counts


def _ssim_of(stats, groups, counts, device):
    """SSIM of a call from its statistics, in float64: the mean over items of the mean over their images."""
    per_image = stats[:, 0] / stats[:, 1]
    item = torch.tensor(groups, device=device)
    per_item = torch.zeros(len(counts), dtype=torch.float64, device=device).index_add_(0, item, per_image)
    return (per_item / torch.tensor(counts, dtype=torch.float64, device=device)).mean()


def native_quality(out, ref):
    """(SSIM, PSNR) as ``training.batch_quality`` computes them, from one ``wn_quality`` call (two launches, no
    per-pixel scratch), as 0-d float64 CUDA tensors.

    ``out``, ``ref``: (N,3,H,W) tensors, one group sharing SSIM's data range: ``ssim`` and ``psnr``.  Or two lists
    of (N_i,3,H_i,W_i) tensors, each item its own group: the mean of the items' SSIMs, and the PSNR of the squared
    error pooled over every element.  Shapes are checked first (ValueError, as ``ssim`` refuses them); CPU tensors
    raise WaterNetLibraryError: there is no CPU path.  SSIM's separable window rounds differently from the 121-tap
    convolution of ``ssim`` (DESIGN.md 4.16 states the bar against float64); the statistics of an item do not depend
    on the other items of the call, bit for bit."""
    eng, _, outs, refs, groups, counts = _native_pairs(out, ref, "native_quality")
    stats = eng.quality(outs, refs, groups)
    s = _ssim_of(stats, groups, counts, eng.device)
    elements = sum(o.numel() for o in outs)
    return s, 10.0 * torch.log10(elements / stats[:, 2].sum())


def ssim_loss(out, ref):
    """``1 - S`` as a 0-d fp32 CUDA tensor, S the SSIM of ``native_quality`` (``ssim`` of a (N,3,H,W) batch, or the
    mean of the items' SSIMs of two lists), computed in float64 and rounded once.  Shapes, devices and refusals are
    those of ``native_quality``.

    When grad is enabled and some ``out`` requires grad, the loss comes from one ``wn_ssim_grad`` call (four
    launches, DESIGN.md 4.17) and autograd keeps only d(loss)/d(out), 12 bytes per pixel: the gradient of torch
    autograd of ``1 - ssim(out, ref)`` (of ``1 - batch_quality(out, ref)[0]`` for lists), the data-range term
    included.  Otherwise it is one ``wn_quality`` call and nothing is kept.  ``ref`` is a constant."""
    eng, items, outs, refs, groups, counts = _native_pairs(out, ref, "ssim_loss")
    if not (torch.is_grad_enabled() and any(o.requires_grad for o, _ in items)):
        stats = eng.quality(outs, refs, groups)
        return (1.0 - _ssim_of(stats, groups, counts, eng.device)).float()
    return _NativeSSIMLoss.apply((eng, items, outs, refs, groups, counts), *[o for o, _ in items])


class _NativeSSIMLoss(torch.autograd.Function):
    """forward: one wn_ssim_grad call with scales -1 / (items x images of the item), so that its gradients are those
    of 1 - S; keeps them, nothing else.  backward: grad_output times each item's gradient."""

    @staticmethod
    def forward(ctx, call, *item_outs):
        eng, items, outs, refs, groups, counts = call
        grads = [torch.empty(o.shape, dtype=torch.float32, device=eng.device) for o in item_outs]
        scales = [-1.0 / (len(counts) * counts[g]) for g in groups]
        stats, _ = eng.ssim_grad(outs, refs, groups, scales, grads=[img for g in grads for img in g])
        ctx.save_for_backward(*grads)
        return (1.0 - _ssim_of(stats, groups, counts, eng.device)).float()

    @staticmethod
    def backward(ctx, grad_output):
        return (None, *(grad_output * g for g in ctx.saved_tensors))
