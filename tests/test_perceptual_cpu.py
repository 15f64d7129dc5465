"""The windowed VGG19 perceptual loss (wn_perceptual_loss) without a GPU: the entry points, the workspace formula and
its rejections, the window rule, and -- in float64 with torch -- that the window decomposition reproduces the
whole-image loss and d(loss)/d(out)."""
import os
import random

import pytest
import torch
import torch.nn as nn

import vgg_reference as V
from conftest import ROOT
from grad_reference import assert_grad_close, grad_error

NEW = ["wn_vgg_pack_weights", "wn_perceptual_loss_workspace_bytes", "wn_perceptual_loss", "wn_debug_vgg_layer"]
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def test_header_declares_and_library_exports_the_new_entry_points(lib):
    from waternet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "waternet_b200.h")).read()
    for name in NEW:
        assert f" {name}(" in header, name
        assert name in _lib.EXPORTED_SYMBOLS
        assert getattr(lib, name) is not None
    assert "#define WN_VGG_NUM_PARAMS 32" in header and _lib.VGG_NUM_PARAMS == 32
    assert lib.wn_abi_version() == _lib.ABI_VERSION


def test_workspace_matches_the_python_restatement(lib):
    from waternet_b200.engine import perceptual_loss_workspace_bytes
    rng = random.Random(5)
    cases = [(1, 16, 16, 0, 0, 0), (3, 37, 53, 16, 16, 0), (2, 300, 500, 48, 32, 0), (4, 1080, 1920, 0, 0, 0),
             (4, 1080, 1920, 998, 998, 0), (1, 3000, 4000, 998, 998, 0), (16, 1080, 1920, 998, 998, 1 << 20),
             (1, 113, 117, 128, 128, 50_000), (65535, 16, 16, 0, 0, 0)]
    cases += [(rng.randint(1, 5), rng.randint(16, 900), rng.randint(16, 900), t, t, rng.choice([0, 30_000, 1 << 21]))
              for t in [rng.randint(1, 400) for _ in range(30)]]
    for args in cases:
        got = lib.wn_perceptual_loss_workspace_bytes(*args)
        assert got > 0 and got == perceptual_loss_workspace_bytes(*args), args


def test_workspace_is_bounded_by_one_pass_whatever_the_image_and_batch_size(lib):
    per_window_pixel = 1900  # act0, two scratch buffers, the 20 saved launch outputs, conv5_4 of ref
    for n, h, w in [(1, 3000, 4000), (16, 1080, 1920), (64, 1080, 1920), (2, 6000, 8000)]:
        ws = lib.wn_perceptual_loss_workspace_bytes(n, h, w, 998, 998, 0)
        windows = n * -(-(h // 16) // 63) * -(-(w // 16) // 63)
        assert ws <= (2 << 20) * per_window_pixel + windows * 16 * 8 + (1 << 20), (n, h, w)


def test_workspace_is_zero_for_rejected_arguments(lib):
    ws = lib.wn_perceptual_loss_workspace_bytes
    assert ws(2, 64, 64, 0, 0, 0) > 0
    assert ws(0, 64, 64, 0, 0, 0) == 0 and ws(-1, 64, 64, 0, 0, 0) == 0      # n <= 0
    assert ws(65536, 16, 16, 0, 0, 0) == 0                                   # n over 65535
    assert ws(1, 15, 64, 0, 0, 0) == 0 and ws(1, 64, 15, 0, 0, 0) == 0        # below 16 x 16
    assert ws(1, 64, 64, 0, 32, 0) == 0 and ws(1, 64, 64, 32, 0, 0) == 0      # one tile side 0
    assert ws(1, 64, 64, -16, -16, 0) == 0                                   # negative tile
    assert ws(1, 64, 64, 0, 0, -1) == 0 and ws(1, 64, 64, 0, 0, (8 << 20) + 1) == 0
    assert ws(1, 64, 64, 0, 0, 8 << 20) > 0
    assert ws(1, 2048, 4096, 0, 0, 0) > 0                                    # one window of exactly 8 Mi pixels
    assert ws(1, 2048, 4112, 0, 0, 0) == 0                                   # a window over the cap ...
    assert ws(1, 2048, 4112, 998, 998, 0) > 0                                # ... that a tile splits
    assert ws(1, 30000, 30000, 998, 998, 0) == 0                             # over the per-image size limit


def test_null_arguments_fail_with_a_message(lib):
    rc = lib.wn_perceptual_loss(None, None, None, None, None, 1, 16, 16, 0, 0, 0, None, None, None, 0, None)
    assert rc == -1 and b"null argument" in lib.wn_last_error()
    assert lib.wn_vgg_pack_weights(None, None, None) == -1


@pytest.mark.parametrize("size", [16, 17, 31, 37, 53, 113, 117, 250, 333, 500, 1080, 1920, 4000])
@pytest.mark.parametrize("tile", [0, 1, 16, 32, 48, 100, 128, 998])
def test_window_rule(size, tile):
    """Starts are multiples of 16, the owned features partition the floor(size / 16) grid in order, and every owned
    feature's 252-pixel support [16 i - 118, 16 i + 133] (clipped to the image) lies in its window."""
    from waternet_b200.engine import VGG_SUPPORT, perceptual_windows
    wins = perceptual_windows(size, tile)
    f = size // 16
    assert wins[0][2] == 0 and wins[-1][3] == f
    for k, (s, e, f0, f1) in enumerate(wins):
        assert s % 16 == 0 and 0 <= s < e <= size and f0 < f1
        if k:
            assert f0 == wins[k - 1][3]
        if tile:
            assert f1 - f0 <= -(-tile // 16)
        assert s <= max(0, 16 * f0 + VGG_SUPPORT[0]) and min(size, 16 * (f1 - 1) + VGG_SUPPORT[1] + 1) <= e
    assert VGG_SUPPORT[1] - VGG_SUPPORT[0] + 1 == 252


def test_support_of_one_feature():
    """[16 i - 118, 16 i + 133]: 4 convolutions at stride 16, a pool, 4 at 8, a pool, 4 at 4, a pool, 2 at 2, a pool,
    2 at 1 (VGG19 features[:-1] read from conv5_4 down)."""
    from waternet_b200.engine import VGG_SUPPORT
    lo, hi = 0, 0  # rows 2^level i + [lo, hi] of the current level
    for level, convs in ((4, 4), (3, 4), (2, 4), (1, 2), (0, 2)):
        lo, hi = lo - convs, hi + convs  # 3 x 3, padding 1
        if level:  # the pool below: rows [2 r, 2 r + 1] of the finer level
            lo, hi = 2 * lo, 2 * hi + 1
    assert (lo, hi) == VGG_SUPPORT


# ---- the decomposition in float64 ------------------------------------------------------------------------------------
def _vgg(widths, seed):
    """VGG19 features[:-1] with channel widths per level ``widths`` (the real one: 64, 128, 256, 512, 512)."""
    g = torch.Generator().manual_seed(seed)
    layers, cin = [], 3
    for level, (convs, width) in enumerate(zip((2, 2, 4, 4, 4), widths)):
        if level:
            layers.append(nn.MaxPool2d(2, 2))
        for _ in range(convs):
            conv = nn.Conv2d(cin, width, 3, padding=1).double()
            with torch.no_grad():
                conv.weight.copy_(torch.randn(conv.weight.shape, generator=g, dtype=torch.float64) * (2.0 / (9 * cin)) ** 0.5)
                conv.bias.copy_(torch.randn(width, generator=g, dtype=torch.float64) * 0.05)
            layers += [conv, nn.ReLU()]
            cin = width
    return nn.Sequential(*layers).eval()


def _norm(x):
    mean = torch.tensor(MEAN, dtype=torch.float32).double().view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=torch.float32).double().view(1, 3, 1, 1)
    return (x - mean) / std


def _whole(vgg, out, ref):
    o = out.clone().requires_grad_(True)
    with torch.no_grad():
        fr = vgg(_norm(ref))
    loss = torch.mean(torch.square(255 * (vgg(_norm(o)) - fr)))
    loss.backward()
    return loss.detach(), o.grad


def _windowed(vgg, out, ref, th, tw, fault=None):
    """The window rule of wn_perceptual_loss: every window's owned features, seeded alone, folded in window order.
    ``fault``: "last_row" (the fold misses each window's last read row), "shift" (it adds a window one row low) or
    "seed_row" (each window also seeds the feature row after its owned ones)."""
    from waternet_b200.engine import perceptual_windows
    n, _, h, w = out.shape
    count = n * vgg[-2].out_channels * (h // 16) * (w // 16)
    loss, grad = torch.zeros((), dtype=torch.float64), torch.zeros_like(out)
    for ys, ye, fy0, fy1 in perceptual_windows(h, th):
        for xs, xe, fx0, fx1 in perceptual_windows(w, tw):
            o = out[:, :, ys:ye, xs:xe].clone().requires_grad_(True)
            with torch.no_grad():
                fr = vgg(_norm(ref[:, :, ys:ye, xs:xe]))
            fo = vgg(_norm(o))
            sy = slice(fy0 - ys // 16, fy1 - ys // 16 + (fault == "seed_row"))
            sx = slice(fx0 - xs // 16, fx1 - xs // 16)
            part = torch.sum(torch.square(255 * (fo[:, :, sy, sx] - fr[:, :, sy, sx]))) / count
            part.backward()
            loss += part.detach()
            if fault == "last_row":
                grad[:, :, ys:ye - 1, xs:xe] += o.grad[:, :, :-1]
            elif fault == "shift":
                grad[:, :, ys + 1:ye, xs:xe] += o.grad[:, :, :-1]
            else:
                grad[:, :, ys:ye, xs:xe] += o.grad
    return loss, grad


# the decomposition depends on the layer structure only: a narrow VGG19 keeps float64 on the CPU fast; the real widths
# run on the small sizes
@pytest.mark.parametrize("shape", [(1, 16, 16), (1, 37, 53), (1, 113, 117), (1, 250, 333), (2, 300, 500)])
@pytest.mark.parametrize("tile", [16, 32, 48, (48, 32), 128])
def test_windows_reproduce_the_whole_image_loss_and_gradient(shape, tile):
    n, h, w = shape
    th, tw = (tile, tile) if isinstance(tile, int) else tile
    widths = (64, 128, 256, 512, 512) if h * w <= 37 * 53 else (4, 8, 8, 8, 8)
    vgg = _vgg(widths, seed=h * 1000 + w)
    g = torch.Generator().manual_seed(7)
    out = torch.rand((n, 3, h, w), generator=g, dtype=torch.float64)
    ref = (out + 0.2 * torch.rand((n, 3, h, w), generator=g, dtype=torch.float64)).clamp(0, 1)
    lw, gw = _whole(vgg, out, ref)
    lt, gt = _windowed(vgg, out, ref, th, tw)
    assert abs(lt - lw) <= 1e-12 * abs(lw)
    assert torch.linalg.vector_norm(gt - gw) <= 1e-12 * torch.linalg.vector_norm(gw)
    assert torch.max(torch.abs(gt - gw)) <= 1e-11 * torch.max(torch.abs(gw))


# ---- the element-wise bar of d(out) ----------------------------------------------------------------------------------
def _conv_pairs(vgg):
    return [(m.weight.detach(), m.bias.detach()) for m in vgg if isinstance(m, nn.Conv2d)]


@pytest.fixture(scope="module")
def chain_case():
    """A narrow VGG19 with nonzero biases on 1 x 250 x 333: the windowed decomposition at tile 48 and the whole-image
    chain R and magnitude M of vgg_reference (the GPU tests' reference, here from a float64 forward)."""
    vgg = _vgg((4, 8, 8, 8, 8), seed=3)
    g = torch.Generator().manual_seed(9)
    out = torch.rand((1, 3, 250, 333), generator=g, dtype=torch.float64)
    ref = (out + 0.2 * torch.rand(out.shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    ws = _conv_pairs(vgg)
    fwd, fref = V.forward_outputs(out, ws), V.forward_outputs(ref, ws)
    seed = V.seed_of(fwd[-1], fref[-1])
    R, M = V.chain(fwd, seed, ws), V.chain(fwd, seed, ws, absolute=True)
    return vgg, out, ref, R, M


def test_the_chain_is_the_whole_image_gradient(chain_case):
    vgg, out, ref, R, M = chain_case
    _, gw = _whole(vgg, out, ref)
    assert_grad_close(gw, R, M, 1e-12, "autograd against the chain")


def test_the_clean_window_fold_passes_the_chain_bar(chain_case):
    vgg, out, ref, R, M = chain_case
    _, gt = _windowed(vgg, out, ref, 48, 48)
    assert_grad_close(gt, R, M, V.TAU_CHAIN["bf16x3"], "windowed d(out)")


@pytest.mark.parametrize("fault", ["last_row", "shift", "seed_row"])
def test_each_fold_fault_fails_the_chain_bar(chain_case, fault):
    """Each fault fails the bar of both arithmetics."""
    vgg, out, ref, R, M = chain_case
    _, gt = _windowed(vgg, out, ref, 48, 48, fault)
    assert grad_error(gt, R, M).max().item() > max(V.TAU_CHAIN.values()), fault


def test_max_pool_picks_the_first_maximum_on_the_cpu():
    V.assert_first_maximum_routing("cpu")


def test_support_mask_is_the_support_of_the_flagged_features():
    from waternet_b200.engine import VGG_SUPPORT
    assert V.SUPPORT == VGG_SUPPORT
    nz = torch.zeros((2, 20, 19), dtype=torch.bool)
    nz[0, 3, 17] = True
    nz[1, 0, 0] = nz[1, 19, 5] = True
    m = V.support_mask(328, 312, nz)[:, 0]
    want = torch.zeros_like(m)
    for n, i, j in nz.nonzero().tolist():
        want[n, max(0, 16 * i - 118):16 * i + 134, max(0, 16 * j - 118):16 * j + 134] = True
    assert torch.equal(m, want)
