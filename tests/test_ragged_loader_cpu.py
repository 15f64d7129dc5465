"""Ragged training batches without a GPU: GpuBatchLoader(ragged=True) yields lists of images in batch order (and
still refuses mixed sizes without it), and the loss of a list batch equals the reference's batch loss on equal sizes.
The loader's engine is replaced by a host stand-in with the same preprocess / resize interface."""
import numpy as np
import pytest
import torch
import torch.nn as nn

SIZES = [(32, 48), (40, 32), (32, 48), (24, 24), (40, 32)]


class _HostEngine:
    """preprocess: x = u/255 and three derived planes; resize_batch: the decoded images are already at size."""
    device = torch.device("cpu")

    def preprocess(self, rgb, tensors=True, images=False):
        x = rgb.permute(0, 3, 1, 2).float() / 255
        return {"x": x, "wb": 1 - x, "gc": x * x, "he": x.flip(1)}

    def resize_batch(self, images, dst_h, dst_w, swap_rb=False):
        for im in images:
            assert im.shape[:2] == (dst_h, dst_w)
        return torch.from_numpy(np.stack(images))


def _loader(dataset, batch_size, ragged, augment=False):
    from waternet_b200.training_utils import GpuBatchLoader
    loader = GpuBatchLoader.__new__(GpuBatchLoader)
    loader.engine = _HostEngine()
    loader.indices = list(range(len(dataset)))
    loader.dataset = dataset
    loader.batch_size = batch_size
    loader.augment = augment
    loader.drop_last = False
    loader.ragged = ragged
    loader.rng = np.random.default_rng(0)
    return loader


class _Files:
    """A file-backed dataset stand-in: decoded(idx) -> (raw, ref, (width, height)) at native size."""

    def __init__(self, sizes):
        from waternet_b200.training_utils import SyntheticUIEB
        self.syn = SyntheticUIEB(len(sizes), sizes=sizes, seed=3)
        self.sizes = sizes

    def __len__(self):
        return len(self.sizes)

    def decoded(self, idx):
        raw, ref = self.syn.pair(idx)
        return raw, ref, (raw.shape[1], raw.shape[0])


@pytest.mark.parametrize("kind", ["pairs", "files"])
def test_ragged_loader_yields_lists_in_batch_order(kind):
    from waternet_b200.training_utils import SyntheticUIEB
    ds = SyntheticUIEB(len(SIZES), sizes=SIZES, seed=3) if kind == "pairs" else _Files(SIZES)
    batches = list(_loader(ds, 4, ragged=True))
    assert len(batches) == 2
    first, second = batches
    for k in ("raw", "wb", "gc", "he", "ref"):
        assert isinstance(first[k], list) and len(first[k]) == 4
    pair = ds.syn.pair if kind == "files" else ds.pair
    for p in range(4):
        raw, ref = pair(p)
        want = torch.from_numpy(raw).permute(2, 0, 1)[None].float() / 255
        assert first["raw"][p].shape == (1, 3) + SIZES[p]
        assert torch.equal(first["raw"][p], want)
        assert torch.equal(first["ref"][p], torch.from_numpy(ref).permute(2, 0, 1)[None].float() / 255)
        assert torch.equal(first["wb"][p], 1 - want)
    # a batch of one size still comes as tensors
    assert torch.is_tensor(second["raw"]) and second["raw"].shape == (1, 3) + SIZES[4]


@pytest.mark.parametrize("kind", ["pairs", "files"])
def test_loader_without_ragged_still_refuses_mixed_sizes(kind):
    from waternet_b200.training_utils import SyntheticUIEB
    ds = SyntheticUIEB(len(SIZES), sizes=SIZES, seed=3) if kind == "pairs" else _Files(SIZES)
    with pytest.raises(ValueError, match="a batch needs one target size"):
        next(iter(_loader(ds, 4, ragged=False)))
    # equal sizes pass either way, as tensors
    same = SyntheticUIEB(4, 32, 48, seed=1)
    for ragged in (False, True):
        b = next(iter(_loader(same, 4, ragged=ragged)))
        assert torch.is_tensor(b["raw"]) and b["raw"].shape == (4, 3, 32, 48)


def test_ragged_loader_augments_each_size_as_a_batch():
    from waternet_b200.training_utils import SyntheticUIEB
    ds = SyntheticUIEB(len(SIZES), sizes=SIZES, seed=3)
    b = next(iter(_loader(ds, 5, ragged=True, augment=True)))
    for p, (h, w) in enumerate(SIZES):  # quarter turns only in pairs for non-square images: the shape is kept
        assert b["raw"][p].shape == (1, 3, h, w)


def test_list_batch_loss_equals_tensor_loss_on_equal_sizes():
    from waternet_b200.training import batch_losses, batch_quality
    torch.manual_seed(0)
    vgg = nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), nn.ReLU(), nn.MaxPool2d(2), nn.Conv2d(8, 4, 3, padding=1))
    out, ref = torch.rand(5, 3, 32, 40, dtype=torch.float64), torch.rand(5, 3, 32, 40, dtype=torch.float64)
    vgg = vgg.double()
    t = batch_losses(vgg, out, ref)
    lst = batch_losses(vgg, list(out.split(1)), list(ref.split(1)))
    for a, b in zip(t, lst):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=0)
    tq = batch_quality(out, ref)
    lq = batch_quality(list(out.split(1)), list(ref.split(1)))
    torch.testing.assert_close(lq[1], tq[1], rtol=1e-12, atol=0)  # PSNR of the pooled MSE
    per_image_ssim = torch.stack([batch_quality(o, r)[0] for o, r in zip(out.split(1), ref.split(1))]).mean()
    torch.testing.assert_close(lq[0], per_image_ssim, rtol=1e-12, atol=0)


def test_list_batch_loss_weights_images_equally():
    from waternet_b200.training import batch_losses
    vgg = nn.Identity()
    out = [torch.zeros(1, 3, 4, 4), torch.zeros(1, 3, 8, 4)]
    ref = [torch.full((1, 3, 4, 4), 1 / 255), torch.full((1, 3, 8, 4), 2 / 255)]
    from waternet_b200.training import perceptual_loss
    loss, perc, mse = batch_losses(vgg, out, ref)
    torch.testing.assert_close(mse, torch.tensor(2.5))  # (1 + 4) / 2, not the pixel-weighted 3.0 of a pooled mean
    percs = [perceptual_loss(vgg, o, r) for o, r in zip(out, ref)]
    torch.testing.assert_close(loss, ((0.05 * percs[0] + 1) + (0.05 * percs[1] + 4)) / 2)
