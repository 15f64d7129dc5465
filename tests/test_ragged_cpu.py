"""Ragged batches (wn_enhance_u8_ragged) without a GPU: the pass plan, the workspace function, the CLI flag."""
import ctypes
import random
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT

BYTES_PER_PIXEL = 1868           # kUmmaBytesPerPixel: one pass of the tensor-core forward
DEFAULT_PASS = 8 << 20           # max_pass_pixels = 0
MODE_DEFAULT, MODE_FP32, MODE_BF16X3 = -1, 0, 1


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def _mix(seed, n=100):
    """A directory-like mix: thumbnails to full HD, plus odd sizes."""
    rng = random.Random(seed)
    common = [(112, 112), (240, 320), (300, 400), (480, 640), (533, 800), (720, 1280), (1080, 1920), (320, 240)]
    odd = [(37, 53), (113, 117), (5, 7), (40, 700), (1, 1)]
    return [rng.choice(odd) if rng.random() < 0.2 else rng.choice(common) for _ in range(n)]


def _ws(lib, sizes, tile=(256, 256), max_pass=0, mode=MODE_DEFAULT):
    n = len(sizes)
    hs = (ctypes.c_int * max(1, n))(*[h for h, _ in sizes])
    ws = (ctypes.c_int * max(1, n))(*[w for _, w in sizes])
    return lib.wn_enhance_ragged_workspace_bytes(hs, ws, n, tile[0], tile[1], max_pass, mode)


def _formula(lib, sizes, tile, max_pass):
    """The workspace the library asks for, from the Python plan: the largest pass x 1868 B + 4096 of slack, the
    per-image LUTs, the descriptor table (images, then windows), and 1024 of alignment slack."""
    from waternet_b200.engine import RAGGED_IMAGE_BYTES, RAGGED_WINDOW_BYTES, ragged_plan
    a256 = lambda v: (v + 255) // 256 * 256  # noqa: E731
    passes = ragged_plan(sizes, *tile, max_pass)
    px = max(len(p["windows"]) * p["slot"][0] * p["slot"][1] for p in passes)
    windows = sum(len(p["windows"]) for p in passes)
    pre = a256(lib.wn_preprocess_workspace_bytes(len(sizes), 8, 8))
    table = a256(a256(len(sizes) * RAGGED_IMAGE_BYTES) + windows * RAGGED_WINDOW_BYTES)
    return px * BYTES_PER_PIXEL + 4096 + pre + table + 1024


PLANS = [(seed, tile, max_pass) for seed in (0, 1, 2)
         for tile, max_pass in [((256, 256), 0), ((256, 256), 1 << 20), ((998, 998), 0), ((128, 96), 300_000)]]


@pytest.mark.parametrize("seed,tile,max_pass", PLANS)
def test_plan_covers_every_image_with_its_tiled_windows(seed, tile, max_pass):
    from waternet_b200.engine import TILE_HALO, ragged_plan, tile_geometry
    sizes = _mix(seed, 40)
    passes = ragged_plan(sizes, *tile, max_pass)
    covered = [np.zeros(s, dtype=np.int32) for s in sizes]
    seen = {i: [] for i in range(len(sizes))}
    for p in passes:
        sh, sw = p["slot"]
        for r in p["windows"]:
            h, w = sizes[r["img"]]
            (ky0, ky1), (kx0, kx1) = r["rows"], r["cols"]
            assert r["vh"] <= sh and r["vw"] <= sw
            assert 0 <= r["ys"] and r["ys"] + r["vh"] <= h and 0 <= r["xs"] and r["xs"] + r["vw"] <= w
            assert r["ys"] <= ky0 < ky1 <= r["ys"] + r["vh"] and r["xs"] <= kx0 < kx1 <= r["xs"] + r["vw"]
            # an inner edge of the valid extent is at least 13 pixels from the kept rectangle
            assert r["ys"] == 0 or ky0 - r["ys"] >= TILE_HALO
            assert r["ys"] + r["vh"] == h or r["ys"] + r["vh"] - ky1 >= TILE_HALO
            assert r["xs"] == 0 or kx0 - r["xs"] >= TILE_HALO
            assert r["xs"] + r["vw"] == w or r["xs"] + r["vw"] - kx1 >= TILE_HALO
            covered[r["img"]][ky0:ky1, kx0:kx1] += 1
            seen[r["img"]].append((r["ys"], r["xs"], r["rows"], r["cols"], r["vh"], r["vw"]))
    assert all((c == 1).all() for c in covered)
    for i, (h, w) in enumerate(sizes):  # exactly the windows the tiled call uses for the image alone
        g = tile_geometry(h, w, *tile)
        want = [(ys, xs, rows, cols, g["win_h"], g["win_w"]) for ys, xs, rows, cols in g["windows"]]
        assert sorted(seen[i]) == sorted(want)


@pytest.mark.parametrize("seed,tile,max_pass", PLANS)
def test_plan_passes_keep_their_limits(seed, tile, max_pass):
    from waternet_b200.engine import ragged_plan
    passes = ragged_plan(_mix(seed, 40), *tile, max_pass)
    for p in passes:
        cnt, slot = len(p["windows"]), p["slot"][0] * p["slot"][1]
        assert p["slot"] == (max(r["vh"] for r in p["windows"]), max(r["vw"] for r in p["windows"]))
        assert cnt <= 65535
        if cnt > 1:
            assert cnt * slot <= (max_pass or DEFAULT_PASS)
            valid = sum(r["vh"] * r["vw"] for r in p["windows"])
            assert 4 * (cnt * slot - valid) <= cnt * slot


def test_plan_mixes_window_sizes_in_a_pass():
    """Tiny and large images together: some pass holds windows of different sizes, so masking is exercised."""
    from waternet_b200.engine import ragged_plan
    sizes = [(5, 7), (37, 53), (113, 117), (112, 112), (300, 520), (40, 700), (1080, 1920)]
    passes = ragged_plan(sizes, 256, 256, 200_000)
    assert len(passes) > 1
    assert any(len({(r["vh"], r["vw"]) for r in p["windows"]}) > 1 for p in passes)
    for seed in range(3):
        assert any(len({(r["vh"], r["vw"]) for r in p["windows"]}) > 1
                   for p in ragged_plan(_mix(seed), 256, 256, 0))


def test_plan_of_many_thumbnails_keeps_the_grid_limit():
    from waternet_b200.engine import ragged_plan
    passes = ragged_plan([(8, 8)] * 70000, 256, 256, 1 << 30)
    assert [len(p["windows"]) for p in passes] == [65535, 70000 - 65535]


@pytest.mark.parametrize("seed,tile,max_pass", PLANS)
def test_workspace_equals_the_formula_of_the_plan(lib, seed, tile, max_pass):
    sizes = _mix(seed, 40)
    assert _ws(lib, sizes, tile, max_pass) == _formula(lib, sizes, tile, max_pass)
    assert _ws(lib, sizes, tile, max_pass, MODE_BF16X3) == _ws(lib, sizes, tile, max_pass)


@pytest.mark.parametrize("size,n", [((5504, 8256), 4), ((1080, 1920), 50), ((112, 112), 500)])
def test_workspace_is_bounded_by_one_pass(lib, size, n):
    """45 MP photos as 1080p frames or thumbnails: one pass + ~84 KB per image + the table."""
    from waternet_b200.engine import RAGGED_IMAGE_BYTES, RAGGED_WINDOW_BYTES, ragged_plan
    sizes = [size] * n
    windows = sum(len(p["windows"]) for p in ragged_plan(sizes, 998, 998))
    per_image = lib.wn_preprocess_workspace_bytes(1, 8, 8)
    assert per_image < 90_000
    got = _ws(lib, sizes, (998, 998))
    bound = DEFAULT_PASS * BYTES_PER_PIXEL + n * per_image + n * RAGGED_IMAGE_BYTES + windows * RAGGED_WINDOW_BYTES \
        + (64 << 10)
    assert 0 < got <= bound
    assert got <= 16e9


def test_bad_arguments_give_no_workspace(lib):
    assert _ws(lib, [(64, 64), (30, 20)]) > 0
    for sizes, tile, max_pass, mode in [
            ([], (256, 256), 0, MODE_DEFAULT),                     # n = 0
            ([(0, 64)], (256, 256), 0, MODE_DEFAULT),              # a size below 1
            ([(64, 64), (64, -3)], (256, 256), 0, MODE_DEFAULT),
            ([(64, 64)], (0, 256), 0, MODE_DEFAULT),               # tile below 1
            ([(64, 64)], (256, -1), 0, MODE_DEFAULT),
            ([(64, 64)], (256, 256), -1, MODE_DEFAULT),            # negative pass size
            ([(64, 64)], (256, 256), 0, MODE_FP32),                # the fp32 CUDA-core mode
            ([(64, 64)], (256, 256), 0, 7),                        # unknown mode
            ([(64, 64), (30000, 30000)], (998, 998), 0, MODE_DEFAULT),  # H x W above 0x7fffffff / 3
            ([(1, 1)] * 65536, (256, 256), 0, MODE_DEFAULT)]:      # n above 65535
        assert _ws(lib, sizes, tile, max_pass, mode) == 0, (len(sizes), sizes[:2], tile, max_pass, mode)
    one = (ctypes.c_int * 1)(64)
    assert lib.wn_enhance_ragged_workspace_bytes(None, one, 1, 256, 256, 0, MODE_DEFAULT) == 0
    assert lib.wn_enhance_ragged_workspace_bytes(one, None, 1, 256, 256, 0, MODE_DEFAULT) == 0


def test_call_with_a_null_handle_fails(lib):
    from waternet_b200 import _lib
    imgs = (_lib.RaggedImage * 1)(_lib.RaggedImage(16, 16, None, 8, 8))
    assert lib.wn_enhance_u8_ragged(None, imgs, 1, 256, 256, 0, MODE_DEFAULT, None, 0, None) != 0
    assert b"null" in lib.wn_last_error()


def test_inference_cli_lists_batch():
    res = subprocess.run([sys.executable, "inference.py", "--help"], cwd=ROOT, capture_output=True, text=True,
                         timeout=120)
    assert res.returncode == 0, res.stderr
    assert "--batch" in res.stdout
