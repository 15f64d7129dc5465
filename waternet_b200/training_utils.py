"""Dataset glue of the reference (``waternet/training_utils.py``) on the CUDA preprocess.

``arr2ten`` / ``ten2arr`` keep the reference's layout-and-scale contract
(``training_utils.py:11-43``: no batch dimension is added to a 3-D array here,
unlike the hubconf variants).  ``UIEBDataset`` keeps the reference's constructor
and item dictionary (``training_utils.py:46-132``); file decoding and resizing
stay with OpenCV (disk-bound glue, out of scope for kernels) while the WB/GC/HE
transform of every item runs on the GPU.  ``SyntheticUIEB`` is the offline
stand-in used by ``train.py --synthetic`` (no UIEB images without network).
"""
from __future__ import annotations

import os
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from .data import transform as preprocess_transform


def arr2ten(arr) -> torch.Tensor:
    """uint8 (N)HWC array -> fp32 (N)CHW tensor scaled to [0,1] (true division by 255)."""
    ten = torch.from_numpy(np.ascontiguousarray(arr)) / 255
    if ten.dim() == 3:
        return ten.permute(2, 0, 1)
    if ten.dim() == 4:
        return ten.permute(0, 3, 1, 2)
    return ten


def ten2arr(ten: torch.Tensor) -> np.ndarray:
    """fp32 (N)CHW tensor -> uint8 (N)HWC array: clip to [0,1], scale by 255, truncate."""
    arr = np.clip(ten.detach().cpu().numpy(), 0, 1)
    arr = (arr * 255).astype(np.uint8)
    if arr.ndim == 3:
        return np.transpose(arr, (1, 2, 0))
    if arr.ndim == 4:
        return np.transpose(arr, (0, 2, 3, 1))
    return arr


class FlipRotate:
    """HorizontalFlip / VerticalFlip / RandomRotate90, each with p=0.5 (training_utils.py:72-78).

    Same call convention as an albumentations Compose: ``t(image=a, mask=b)`` ->
    ``{"image": a', "mask": b'}``; seeded so that runs are reproducible.
    """

    def __init__(self, seed: Optional[int] = None):
        self.rng = np.random.default_rng(seed)

    def __call__(self, image, mask):
        if self.rng.random() < 0.5:
            image, mask = image[:, ::-1], mask[:, ::-1]
        if self.rng.random() < 0.5:
            image, mask = image[::-1], mask[::-1]
        if self.rng.random() < 0.5:
            k = int(self.rng.integers(0, 4))
            image, mask = np.rot90(image, k), np.rot90(mask, k)
        return {"image": np.ascontiguousarray(image), "mask": np.ascontiguousarray(mask)}


def _item(raw_im: np.ndarray, ref_im: np.ndarray):
    wb, gc, he = preprocess_transform(raw_im)
    return {"raw": arr2ten(raw_im), "wb": arr2ten(wb), "gc": arr2ten(gc), "he": arr2ten(he), "ref": arr2ten(ref_im)}


class UIEBDataset(torch.utils.data.Dataset):
    """Paired raw/reference PNG folders (same file names in both)."""

    def __init__(self, raw_dir, ref_dir, im_height: Optional[int] = None, im_width: Optional[int] = None,
                 transform=None):
        raw_names = sorted(p.name for p in Path(raw_dir).glob("*.png"))
        ref_names = sorted(p.name for p in Path(ref_dir).glob("*.png"))
        assert set(raw_names) == set(ref_names)
        self.transform = transform if transform is not None else FlipRotate()
        self.raw_dir, self.ref_dir = Path(raw_dir), Path(ref_dir)
        self.im_fns = raw_names
        self.im_height, self.im_width = im_height, im_width

    def __len__(self):
        return len(self.im_fns)

    def decoded(self, idx):
        """The two files of item ``idx`` as decoded by ``cv2.imread`` (BGR uint8, native size) and the
        ``(width, height)`` the reference resizes them to (training_utils.py:94-103)."""
        import cv2  # file decode only
        raw_im = cv2.imread(os.fspath(self.raw_dir / self.im_fns[idx]))
        ref_im = cv2.imread(os.fspath(self.ref_dir / self.im_fns[idx]))
        if self.im_width is not None and self.im_height is not None:
            size = (self.im_width, self.im_height)
        else:  # multiple of 32 for VGG; the reference swaps the axis names here (training_utils.py:100-103)
            size = (int(raw_im.shape[0] / 32) * 32, int(raw_im.shape[1] / 32) * 32)
        return raw_im, ref_im, size

    def pair(self, idx):
        """Decoded, resized RGB uint8 (raw, ref) arrays of item ``idx`` -- no augmentation, no preprocess
        (the per-item CPU path; ``GpuBatchLoader`` resizes on the device instead)."""
        import cv2
        raw_im, ref_im, size = self.decoded(idx)
        raw_im = cv2.cvtColor(cv2.resize(raw_im, size), cv2.COLOR_BGR2RGB)
        ref_im = cv2.cvtColor(cv2.resize(ref_im, size), cv2.COLOR_BGR2RGB)
        return raw_im, ref_im

    def __getitem__(self, idx):
        raw_im, ref_im = self.pair(idx)
        if self.transform is not None:
            t = self.transform(image=raw_im, mask=ref_im)
            raw_im, ref_im = t["image"], t["mask"]
        return _item(raw_im, ref_im)


class SyntheticUIEB(torch.utils.data.Dataset):
    """UIEB-shaped synthetic pairs: a smooth scene (reference) and a blue-green degraded copy (raw).  ``sizes``: a
    list of (h, w); item idx then has size sizes[idx % len(sizes)] instead of im_height x im_width (a dataset whose
    items keep their own sizes)."""

    def __init__(self, length: int = 890, im_height: int = 112, im_width: int = 112, seed: int = 0, transform=None,
                 sizes=None):
        self.length, self.h, self.w, self.seed = length, im_height, im_width, seed
        self.transform = transform
        self.sizes = list(sizes) if sizes else None

    def __len__(self):
        return self.length

    def _scene(self, idx):
        h, w = self.sizes[idx % len(self.sizes)] if self.sizes else (self.h, self.w)
        rng = np.random.default_rng(self.seed * 100003 + idx)
        coarse = rng.random((h // 8 + 2, w // 8 + 2, 3))
        ref = np.kron(coarse, np.ones((8, 8, 1)))[:h, :w]
        ref = (ref * 255).astype(np.uint8)
        cast = np.array([0.35, 0.8, 0.9])
        raw = (ref.astype(np.float64) * cast * (0.6 + 0.4 * rng.random())).astype(np.uint8)
        raw = np.maximum(raw, 1)
        return raw, ref

    def pair(self, idx):
        return self._scene(idx)

    def __getitem__(self, idx):
        raw_im, ref_im = self._scene(idx)
        if self.transform is not None:
            t = self.transform(image=raw_im, mask=ref_im)
            raw_im, ref_im = t["image"], t["mask"]
        return _item(raw_im, ref_im)


class GpuBatchLoader:
    """Training batches assembled on the GPU (SURVEY.md section 8f.3).

    The reference's loop is data-loading bound: every item runs ``transform`` and four ``arr2ten`` on
    the CPU in the main process (``training_utils.py:89-132``, ``train.py:234``).  Here a batch of
    uint8 (raw, ref) pairs goes to the device once (file-backed datasets: at native size, resized there by ONE
    batched ``wn_resize_u8`` with cv2's exact INTER_LINEAR arithmetic); the flip / rot90 augmentation (same p=0.5 choices
    as ``training_utils.py:72-78``, applied identically to raw and ref) and ONE batched
    ``wn_preprocess_u8`` produce the five fp32 tensors of the reference's item dictionary, already
    on the device.  ``dataset`` needs ``__len__`` and ``pair(idx) -> (raw_u8, ref_u8)`` (both
    datasets of this module have it); ``torch.utils.data.Subset`` views are accepted.

    ``ragged``: a batch whose items have different sizes (a dataset without im_height / im_width, which keeps every
    item at its own size) comes as five lists ``raw, wb, gc, he, ref`` of (1,3,H_i,W_i) tensors in batch order, for
    ``WaterNet.forward_many``.  Each distinct size is resized, augmented and preprocessed as one batch (a quarter
    turn is applied to a non-square item only in pairs, as in a tensor batch).  A batch of one size still comes as
    tensors.  Without it (the default) such a batch raises.
    """

    def __init__(self, dataset, batch_size: int, device=None, augment: bool = True, seed: Optional[int] = None,
                 drop_last: bool = False, ragged: bool = False):
        from .engine import get_engine
        self.engine = get_engine(device)
        self.indices = list(range(len(dataset)))
        while isinstance(dataset, torch.utils.data.Subset):  # unwrap random_split views
            self.indices = [dataset.indices[i] for i in self.indices]
            dataset = dataset.dataset
        self.dataset = dataset
        self.batch_size = batch_size
        self.augment = augment
        self.drop_last = drop_last
        self.ragged = ragged
        self.rng = np.random.default_rng(seed)

    def __len__(self):
        n = len(self.indices)
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def _augment(self, raw: torch.Tensor, ref: torch.Tensor):
        """Per-sample HorizontalFlip / VerticalFlip / RandomRotate90 (p=0.5 each) on NHWC uint8 batches."""
        square = raw.shape[1] == raw.shape[2]
        outs_raw, outs_ref = [], []
        for i in range(raw.shape[0]):
            a, b = raw[i], ref[i]
            if self.rng.random() < 0.5:
                a, b = a.flip(1), b.flip(1)
            if self.rng.random() < 0.5:
                a, b = a.flip(0), b.flip(0)
            if self.rng.random() < 0.5:
                k = int(self.rng.integers(0, 4))
                if not square:
                    k = (k // 2) * 2  # a quarter turn would change the shape inside a batch
                a, b = torch.rot90(a, k, (0, 1)), torch.rot90(b, k, (0, 1))
            outs_raw.append(a)
            outs_ref.append(b)
        return torch.stack(outs_raw).contiguous(), torch.stack(outs_ref).contiguous()

    def __iter__(self):
        dev = self.engine.device
        for start in range(0, len(self.indices), self.batch_size):
            idx = self.indices[start:start + self.batch_size]
            if self.drop_last and len(idx) < self.batch_size:
                break
            if hasattr(self.dataset, "decoded"):
                # file-backed dataset: cv2.imread on the host, then ONE batched bilinear resize + BGR->RGB on the
                # device (wn_resize_u8, bit-exact cv2.resize arithmetic) per target size instead of 2 x batch
                # cv2.resize calls
                items = [self.dataset.decoded(i) for i in idx]
                groups = self._groups([(it[2][1], it[2][0]) for it in items])
                batches = []
                for (dh, dw), pos in groups:
                    raw = self.engine.resize_batch([items[p][0] for p in pos], dh, dw, swap_rb=True)
                    ref = self.engine.resize_batch([items[p][1] for p in pos], dh, dw, swap_rb=True)
                    batches.append((pos, raw, ref))
            else:
                pairs = [self.dataset.pair(i) for i in idx]
                groups = self._groups([p[0].shape[:2] for p in pairs])
                batches = []
                for _, pos in groups:
                    raw = torch.from_numpy(np.stack([pairs[p][0] for p in pos])).to(dev, non_blocking=True)
                    ref = torch.from_numpy(np.stack([pairs[p][1] for p in pos])).to(dev, non_blocking=True)
                    batches.append((pos, raw, ref))
            done = [(pos, self._tensors(raw, ref)) for pos, raw, ref in batches]
            if len(done) == 1:
                yield done[0][1]
                continue
            out = {k: [None] * len(idx) for k in ("raw", "wb", "gc", "he", "ref")}
            for pos, t in done:
                for j, p in enumerate(pos):
                    for k in out:
                        out[k][p] = t[k][j:j + 1]
            yield out

    def _groups(self, sizes):
        """[((h, w), [positions in the batch])] in order of first appearance; more than one size only if ragged."""
        groups = {}
        for p, s in enumerate(sizes):
            groups.setdefault(tuple(int(v) for v in s), []).append(p)
        if len(groups) > 1 and not self.ragged:
            raise ValueError("a batch needs one target size: give the dataset im_height / im_width, or pass "
                             "ragged=True for batches of lists")
        return list(groups.items())

    def _tensors(self, raw: torch.Tensor, ref: torch.Tensor):
        """Augment and preprocess one batch of equally sized NHWC uint8 pairs -> the five fp32 tensors."""
        if self.augment:
            raw, ref = self._augment(raw, ref)
        pre = self.engine.preprocess(raw, tensors=True, images=False)
        # u/255 must be the true fp32 quotient (arr2ten): torch's CUDA "tensor / scalar" multiplies by a
        # reciprocal, so the reference image goes through the library's exact table as well
        ref_t = self.engine.preprocess(ref, tensors=True, images=False)["x"]
        return {"raw": pre["x"], "wb": pre["wb"], "gc": pre["gc"], "he": pre["he"], "ref": ref_t}
