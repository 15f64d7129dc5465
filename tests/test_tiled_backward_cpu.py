"""Windowed recompute backward (wn_backward_tiled) without a GPU: the workspace bound, the rejected arguments, the
covering-window rule the input gradients are folded by, and the ``grad_tile`` attribute and ``--grad-tile`` flag."""
import copy
import io
import os
import subprocess
import sys

import pytest
import torch

TRAIN_BYTES_PER_PIXEL = 5616                    # kTrainBytesPerPixel: every activation and gradient buffer of a pass
DEFAULT_PASS = 2 << 20                          # max_pass_pixels = 0
MAX_PASS = 8 << 20                              # kTrainMaxPixels
DENSE_BYTES = 49 * 128 * 128 * 4                # kDenseBytes: one layer's weight gradient, dense
PARTIAL_BYTES = 192 * 512 * 128 * 4             # kPartialBytes: per-CTA partial sums of the weight-gradient GEMMs
PARAM_BYTES = 1_200_000 * 4                     # scratch copy of the 34 parameter gradients (~1.1 M floats)
FIXED = DENSE_BYTES + PARTIAL_BYTES + PARAM_BYTES + (64 << 10)
SIZES = [(64, 64), (300, 520), (1080, 1920), (2160, 3840), (4320, 7680), (5504, 8256), (20000, 30000)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.mark.parametrize("n", [1, 16])
@pytest.mark.parametrize("h,w", SIZES)
def test_workspace_is_bounded_by_one_pass(lib, n, h, w):
    for max_pass in (0, 1 << 20, 4 << 20, MAX_PASS):
        got = lib.wn_backward_tiled_workspace_bytes(n, h, w, 998, 998, max_pass)
        bound = (max_pass or DEFAULT_PASS) * TRAIN_BYTES_PER_PIXEL + FIXED
        assert 0 < got <= bound, (n, h, w, max_pass, got, bound)


def test_workspace_does_not_grow_with_the_image(lib):
    sizes = [lib.wn_backward_tiled_workspace_bytes(1, h, w, 998, 998, 0) for h, w in SIZES[2:]]
    assert max(sizes) <= DEFAULT_PASS * TRAIN_BYTES_PER_PIXEL + FIXED
    assert lib.wn_backward_tiled_workspace_bytes(16, 1080, 1920, 998, 998, 0) <= max(sizes) * 1.1


def test_45_mp_photo_needs_about_10_gb(lib):
    got = lib.wn_backward_tiled_workspace_bytes(1, 5504, 8256, 998, 998, 0)
    assert 2 * 944 * 944 * TRAIN_BYTES_PER_PIXEL < got <= 2 * 944 * 944 * TRAIN_BYTES_PER_PIXEL + FIXED  # 2 windows
    assert 9.5e9 < got < 10.5e9
    assert lib.wn_train_workspace_bytes(1, 5504, 8256) > 250e9  # what keeping every activation would take


def test_bad_arguments_give_no_workspace(lib):
    fn = lib.wn_backward_tiled_workspace_bytes
    assert fn(1, 64, 64, 32, 32, 0) > 0
    assert fn(1, 64, 64, 32, 32, MAX_PASS) > 0
    assert fn(1, 2048, 4096, 4096, 4096, 0) > 0  # one 8 Mi-pixel window
    for args in [(0, 64, 64, 32, 32, 0), (-1, 64, 64, 32, 32, 0), (1, 0, 64, 32, 32, 0), (1, 64, -1, 32, 32, 0),
                 (1, 64, 64, 0, 32, 0), (1, 64, 64, 32, -5, 0), (1, 64, 64, 32, 32, -1),
                 (1, 64, 64, 32, 32, MAX_PASS + 1), (65536, 64, 64, 32, 32, 0),
                 (1, 30000, 30000, 998, 998, 0),  # over the size limit (~715 Mpx)
                 (1, 2049, 4096, 4096, 4096, 0),  # a window of more than 8 Mi pixels
                 (1, 3000, 4000, 3000, 4000, 0)]:
        assert fn(*args) == 0, args


def test_null_arguments_fail_with_a_message(lib):
    assert lib.wn_backward_tiled(None, None, None, None, None, None, None, None, None, 1, 64, 64, 32, 32, 0, None, 0,
                                 None) != 0
    assert b"wn_backward_tiled: null" in lib.wn_last_error()


def _brute_force(g, y, x):
    return sorted((i, j) for i in range(g["ny"]) for j in range(g["nx"])
                  for ys, xs in [g["windows"][i * g["nx"] + j][:2]]
                  if ys <= y < ys + g["win_h"] and xs <= x < xs + g["win_w"])


@pytest.mark.parametrize("h,w,tile", [(5, 7, (1, 1)), (37, 53, (8, 8)), (97, 131, (16, 16)), (97, 131, (32, 32)),
                                      (45, 70, (45, 16)), (60, 41, (7, 19)), (30, 30, (64, 64)), (30, 30, (30, 30)),
                                      (200, 90, (26, 27)), (130, 140, (40, 100))])
def test_covering_windows_match_brute_force(h, w, tile):
    from waternet_b200.engine import covering_windows, tile_geometry
    g = tile_geometry(h, w, *tile)
    counts = set()
    for y in range(h):
        for x in range(w):
            rows, cols = covering_windows(g, y, x)
            got = [(i, j) for i in rows for j in cols]
            assert got == _brute_force(g, y, x), (y, x, got)
            counts.add(len(rows))
    if tile[0] == 1:
        assert max(counts) == g["ny"]  # tile 1 on a small image: every window is the whole image


def test_grad_tile_defaults_to_none_and_survives_deepcopy_and_pickling():
    from oracle import forward as ofw
    from waternet_b200.net import WaterNet
    plain = WaterNet()
    m = WaterNet(grad_tile=(64, 96))
    m.load_state_dict(ofw.synthetic_state_dict(0))
    assert plain.grad_tile is None and m.grad_tile == (64, 96) and m.tile is None
    assert list(m.state_dict().keys()) == list(plain.state_dict().keys())
    assert copy.deepcopy(m).grad_tile == (64, 96)
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert again.grad_tile == (64, 96)
    del again.__dict__["grad_tile"]  # a model pickled before the attribute existed
    assert again.grad_tile is None


def test_grad_tile_with_the_fp32_precision_is_refused():
    from waternet_b200.net import WaterNet
    with pytest.raises(ValueError, match="tensor cores"):
        WaterNet(precision="fp32", grad_tile=64)
    with pytest.raises(ValueError):
        WaterNet(grad_tile=0)
    m = WaterNet(precision="fp32")
    m.grad_tile = 64
    with pytest.raises(ValueError, match="tensor cores"):
        m(*[torch.rand(1, 3, 8, 8, requires_grad=True) for _ in range(4)])


def test_train_help_lists_grad_tile():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "train.py"), "--help"], capture_output=True, text=True,
                         cwd=ROOT)
    assert res.returncode == 0, res.stderr
    assert "--grad-tile" in res.stdout
