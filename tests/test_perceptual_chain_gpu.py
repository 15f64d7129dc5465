"""d(loss)/d(out) of the native perceptual loss on the GPU, element by element, at every call form.

Every window's share of d(out) passes through activations that are bit for bit the whole-image ones (DESIGN.md 4.12,
window rule), so one float64 chain from the GPU's whole-image seed, ReLU' masks and pool routes (vgg_reference.chain)
is the reference of the one-window call, of every tile and of every split into passes: |G - R| <= TAU_CHAIN M
element by element, M the same chain of |seed| through |W|.  Where M is 0 the bar asks for exactly 0.  A fold that drops or
shifts a window's rows, folds into the wrong image or counts a feature twice moves elements by a share of their own
M, which a norm-wise comparison of whole tensors hides.  Probe pairs (ref == out except for 3 x 3 patches) add
exactness: the seed is 0 at every feature whose support misses the patches, and d(out) is 0.0 outside the support of
the features it seeds.  Both arithmetics (bf16x3, bf16) and both weight sets of vgg_reference."""
import functools
import os

import pytest
import torch

import bf16_replay as rp
import vgg_reference as V
from grad_reference import assert_grad_close

pytestmark = pytest.mark.gpu

MODES = ("bf16x3", "bf16")
SHAPE = (3, 320, 320)
# at tile 16 the middle windows of a 320-pixel axis (k = 8..11) are one class of 272 x 272 pixels, 4 x 4 per image:
# passes of 2 of them split a window row, of 3 cross window rows inside an image, of 6 cross images
CLASS_PX = 272 * 272
SPLITS = {"row": 2 * CLASS_PX, "image": 3 * CLASS_PX, "images": 6 * CLASS_PX}
CALLS = [(None, 0), (16, 0), (32, 0), (48, 0), ((48, 32), 0), (128, 0)] + [(16, m) for m in SPLITS.values()]
CALL_IDS = ["one-window", "t16", "t32", "t48", "t48x32", "t128"] + [f"t16-split-{k}" for k in SPLITS]
PROBE_SHAPE = (2, 328, 312)  # rows 320..327 and columns 304..311 lie beyond 16 F
# image corners, a patch whose last nonzero feature row (8) is the last owned row of a 48-pixel window, a window corner
# of tiles 16 / 32 / 48 (x = 96, y = 144), and rows beyond 16 F
PROBES = [(0, 0, 0), (0, 325, 200), (1, 10, 10), (1, 142, 94), (1, 325, 309)]
PROBE_TILES = [None, 16, 48, (48, 32), 128]
LOSS_REL = 2.0 ** -22


def _mode(name):
    from waternet_b200 import _lib
    return {"bf16x3": _lib.MODE_BF16X3, "bf16": _lib.MODE_BF16}[name]


def _report(name, value):
    path = os.environ.get("WN_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(f"chain {name} {value:.3e}\n")


@functools.lru_cache(maxsize=None)
def _model(wset):
    return V.perceptual_model(wset)


@functools.lru_cache(maxsize=None)
def _whole(mode, wset, probe):
    """(out, ref, R, M, loss from the features, seed) of one mode, weight set and pair: the GPU's whole-image forward,
    seed and features, the float64 chain from them (bf16: with the bf16-rounded weights the launches read)."""
    out, ref = V.probe_pair(*PROBE_SHAPE, PROBES) if probe else V.noise_pair(*SHAPE, seed=31)
    out, ref = out.cuda(), ref.cuda()
    eng, tm = _model(wset)._vgg_engine(out), _mode(mode)
    fwd = [eng.debug_vgg_layer(out, k, train_mode=tm).double() for k in range(20)]
    fr = eng.debug_vgg_layer(ref, 19, train_mode=tm).double()
    seed = eng.debug_vgg_layer(out, 21, ref=ref, train_mode=tm).double()
    ws = V.weights(wset)
    if mode == "bf16":
        ws = [(rp._bf16(w.double()), b) for w, b in ws]
    R, M = V.chain(fwd, seed, ws), V.chain(fwd, seed, ws, absolute=True)
    loss = torch.square(255.0 * (fwd[19] - fr)).sum().item() / fr.numel()
    return out, ref, R, M, loss, seed


def _check_call(mode, wset, probe, tile, mpp=0):
    out, ref, R, M, want, _ = _whole(mode, wset, probe)
    loss, G = _model(wset)._vgg_engine(out).perceptual_loss(out, ref, tile=tile, want_grad=True, max_pass_pixels=mpp,
                                                            train_mode=_mode(mode))
    assert abs(loss.item() - want) <= LOSS_REL * want, (loss.item(), want)
    worst = assert_grad_close(G, R, M, V.TAU_CHAIN[mode], f"d(out) of tile {tile}, max_pass_pixels {mpp}")
    _report(f"{mode} {wset} {'probe' if probe else 'noise'} tile={tile} mpp={mpp}", worst)
    return G


def test_bars_are_under_their_ceilings():
    for mode in MODES:
        assert V.TAU_CHAIN[mode] <= V.CHAIN_CEILING[mode], mode


def _pass_kinds(n, h, w, tile, mpp):
    """What the passes of wn_perceptual_loss's plan span: "row" (part of one window row), "image" (window rows of one
    image) or "images" -- restated from vgg_plan from the window rule of engine.perceptual_windows."""
    from waternet_b200.engine import VGG_PASS_PIXELS, perceptual_windows

    def runs(size):
        out = []
        for s, e, _, _ in perceptual_windows(size, tile):
            if out and out[-1][1] == e - s:
                out[-1][0] += 1
            else:
                out.append([1, e - s])
        return out
    kinds = set()
    for nky, wh in runs(h):
        for nkx, ww in runs(w):
            per = min(65535, max(1, (mpp or VGG_PASS_PIXELS) // (wh * ww)))
            total = n * nky * nkx
            for w0 in range(0, total, per):
                j = list(range(w0, min(total, w0 + per)))
                imgs = {i // (nky * nkx) for i in j}
                rows = {i // nkx for i in j}
                if len(imgs) > 1:
                    kinds.add("images")
                elif len(rows) > 1 and len(j) < nky * nkx:
                    kinds.add("image")
                elif len(j) < nkx:
                    kinds.add("row")
    return kinds


@pytest.mark.parametrize("split", SPLITS)
def test_the_pass_splits_span_what_they_name(split):
    assert split in _pass_kinds(*SHAPE, 16, SPLITS[split])


@pytest.mark.parametrize("call", CALLS, ids=CALL_IDS)
@pytest.mark.parametrize("wset", V.WEIGHT_SETS)
@pytest.mark.parametrize("mode", MODES)
def test_every_call_against_the_whole_image_chain(mode, wset, call):
    """d(out) of the call within TAU_CHAIN M of the whole-image chain element by element; the loss the float64 sum
    over the GPU's own conv5_4 features within 2^-22."""
    tile, mpp = call
    _check_call(mode, wset, False, tile, mpp)


@pytest.mark.parametrize("tile", PROBE_TILES, ids=[str(t) for t in PROBE_TILES])
@pytest.mark.parametrize("wset", V.WEIGHT_SETS)
@pytest.mark.parametrize("mode", MODES)
def test_probes_are_exact_outside_their_support(mode, wset, tile):
    """The seed is exactly 0 at every feature whose 252-pixel support misses every patch; d(out) is exactly 0.0
    outside the support of the nonzero seeded features, and within the chain bar everywhere."""
    n, h, w = PROBE_SHAPE
    *_, seed = _whole(mode, wset, True)
    touched = torch.zeros((n, h, w), dtype=torch.bool, device="cuda")
    for i, y, x in PROBES:
        touched[i, y:y + 3, x:x + 3] = True
    reach = V.support_mask(h, w, torch.ones((n, h // 16, w // 16), dtype=torch.bool, device="cuda"))
    assert reach.all()  # every pixel of these sizes reaches some feature
    # features whose support holds a patch pixel: the support rule read the other way
    fy = torch.arange(h // 16, device="cuda")
    fx = torch.arange(w // 16, device="cuda")
    near = torch.zeros((n, h // 16, w // 16), dtype=torch.bool, device="cuda")
    for i, y, x in PROBES:
        ry = (16 * fy + V.SUPPORT[0] <= y + 2) & (16 * fy + V.SUPPORT[1] >= y)
        rx = (16 * fx + V.SUPPORT[0] <= x + 2) & (16 * fx + V.SUPPORT[1] >= x)
        near[i] |= ry[:, None] & rx[None, :]
    nonzero = seed.ne(0).any(1)
    assert not (nonzero & ~near).any(), "a seed outside the reach of every patch"
    assert nonzero.any()
    G = _check_call(mode, wset, True, tile)
    inside = V.support_mask(h, w, nonzero).expand_as(G)
    assert (~inside).any(), "the probes leave no pixel outside the support"
    assert torch.count_nonzero(G[~inside]) == 0, "d(out) is not 0 outside the support of the seeded features"
