"""Tiled enhance (wn_enhance_u8_tiled) without a GPU: the workspace bound, the window rule, the CLI flag."""
import subprocess
import sys

import pytest

from conftest import ROOT

BYTES_PER_PIXEL = 1868           # kUmmaBytesPerPixel: one pass of the tensor-core forward
DEFAULT_PASS = 8 << 20           # max_pass_pixels = 0
SLACK = 64 << 10
MODE_DEFAULT, MODE_FP32, MODE_BF16X3 = -1, 0, 1


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def _pre_bytes_per_image(lib):
    return lib.wn_preprocess_workspace_bytes(1, 8, 8)  # per-image LUTs and histograms; independent of the size


SIZES = [(64, 64), (300, 520), (1080, 1920), (2160, 3840), (4000, 6000), (4320, 7680), (5504, 8256), (20000, 30000)]


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("h,w", SIZES)
def test_tiled_workspace_is_bounded_by_one_pass(lib, n, h, w):
    for max_pass in (0, 1 << 20, 3 << 20, 32 << 20):
        got = lib.wn_enhance_tiled_workspace_bytes(n, h, w, 998, 998, max_pass, MODE_DEFAULT)
        bound = (max_pass or DEFAULT_PASS) * BYTES_PER_PIXEL + n * _pre_bytes_per_image(lib) + SLACK
        assert 0 < got <= bound, (n, h, w, max_pass, got, bound)
        assert lib.wn_enhance_tiled_workspace_bytes(n, h, w, 998, 998, max_pass, MODE_BF16X3) == got


@pytest.mark.parametrize("h,w", [(3000, 4195), (4000, 6000), (4320, 7680), (5504, 8256), (20000, 30000)])
def test_tiled_workspace_below_untiled_from_12_mi_pixels(lib, h, w):
    assert h * w >= 12 << 20
    assert (lib.wn_enhance_tiled_workspace_bytes(1, h, w, 998, 998, 0, MODE_DEFAULT)
            < lib.wn_enhance_workspace_bytes(1, h, w, MODE_DEFAULT))


def test_45_mp_photo_fits_in_16_gb(lib):
    got = lib.wn_enhance_tiled_workspace_bytes(1, 5504, 8256, 998, 998, 0, MODE_DEFAULT)
    assert got <= 16e9
    assert lib.wn_enhance_workspace_bytes(1, 5504, 8256, MODE_DEFAULT) > 80e9  # what the untiled call would need


@pytest.mark.parametrize("h,w,windows,win,recompute", [
    (2160, 3840, 12, (986, 746), 1.064),
    (4320, 7680, 40, (986, 890), 1.058),
    (5504, 8256, 54, (944, 944), 1.059),
])
def test_window_rule_and_workspace_formula(lib, h, w, windows, win, recompute):
    """The worked numbers of the design: window count and size, recompute factor, and the workspace the library
    asks for = (windows per pass) x window x 1868 B + the per-image LUTs + fixed slack."""
    from waternet_b200.engine import tile_geometry
    g = tile_geometry(h, w, 998, 998)
    assert len(g["windows"]) == windows and (g["win_w"], g["win_h"]) == win  # window as width x height
    assert round(windows * win[0] * win[1] / (h * w), 3) == recompute
    per_pass = min(DEFAULT_PASS // (win[0] * win[1]), windows)
    pre = (lib.wn_preprocess_workspace_bytes(1, h, w) + 255) // 256 * 256
    assert lib.wn_enhance_tiled_workspace_bytes(1, h, w, 998, 998, 0, MODE_DEFAULT) == \
        per_pass * win[0] * win[1] * BYTES_PER_PIXEL + 4096 + pre + 1024


@pytest.mark.parametrize("h,w,th,tw", [(2160, 3840, 998, 998), (300, 520, 64, 96), (37, 53, 256, 256),
                                        (40, 700, 128, 128), (113, 117, 32, 32), (50, 70, 8, 8), (1, 1, 1, 1),
                                        (10, 13, 3, 4)])
def test_windows_cover_the_image_and_keep_the_halo(h, w, th, tw):
    """Kept rectangles tile the image exactly; every window lies inside the image, has the call's size, and each
    window edge inside the image is at least 13 pixels from the kept rectangle."""
    from waternet_b200.engine import TILE_HALO, tile_geometry
    g = tile_geometry(h, w, th, tw)
    assert g["th"] <= th and g["tw"] <= tw
    covered = [[0] * w for _ in range(h)]
    for ys, xs, (ky0, ky1), (kx0, kx1) in g["windows"]:
        assert 0 <= ys and ys + g["win_h"] <= h and 0 <= xs and xs + g["win_w"] <= w
        assert ky0 < ky1 and kx0 < kx1
        assert ys == 0 or ky0 - ys >= TILE_HALO
        assert xs == 0 or kx0 - xs >= TILE_HALO
        assert ys + g["win_h"] == h or ys + g["win_h"] - ky1 >= TILE_HALO
        assert xs + g["win_w"] == w or xs + g["win_w"] - kx1 >= TILE_HALO
        for y in range(ky0, ky1):
            for x in range(kx0, kx1):
                covered[y][x] += 1
    assert all(c == 1 for row in covered for c in row)


def test_bad_arguments_give_no_workspace(lib):
    ok = lib.wn_enhance_tiled_workspace_bytes(1, 64, 64, 32, 32, 0, MODE_DEFAULT)
    assert ok > 0
    for args in [(0, 64, 64, 32, 32, 0, MODE_DEFAULT), (1, 0, 64, 32, 32, 0, MODE_DEFAULT),
                 (1, 64, -1, 32, 32, 0, MODE_DEFAULT), (1, 64, 64, 0, 32, 0, MODE_DEFAULT),
                 (1, 64, 64, 32, -5, 0, MODE_DEFAULT), (1, 64, 64, 32, 32, -1, MODE_DEFAULT),
                 (1, 64, 64, 32, 32, 0, MODE_FP32), (1, 64, 64, 32, 32, 0, 7),
                 (1, 30000, 30000, 998, 998, 0, MODE_DEFAULT)]:  # over the preprocess limit (~715 Mpx)
        assert lib.wn_enhance_tiled_workspace_bytes(*args) == 0, args
    assert lib.wn_enhance_u8_tiled(None, None, None, None, 1, 64, 64, 32, 32, 0, MODE_DEFAULT, None, 0, None) != 0
    assert b"null" in lib.wn_last_error()


def test_inference_cli_lists_tile():
    res = subprocess.run([sys.executable, "inference.py", "--help"], cwd=ROOT, capture_output=True, text=True,
                         timeout=120)
    assert res.returncode == 0, res.stderr
    assert "--tile" in res.stdout
