"""The windowed recompute backward of a ragged batch (wn_backward_ragged_tiled) without a GPU: the entry points, the
workspace bound and its rejections, and the plan property the input-gradient fold relies on."""
import ctypes
import os
import random

import pytest

from conftest import ROOT

TRAIN_BYTES_PER_PIXEL = 5616  # kTrainBytesPerPixel: every activation and gradient buffer of a pass
TRAIN_MAX = 8 << 20           # pixels of one training pass
DEFAULT_PASS = 2 << 20        # max_pass_pixels = 0
PACK_IN_ARGS_BYTES = 160      # csrc/common.cuh PackInArgs: one per image
RAGGED_GRADS_BYTES = 40       # csrc/conv_bwd.cu RaggedGrads: one per image
NEW = ["wn_backward_ragged_tiled_workspace_bytes", "wn_backward_ragged_tiled"]


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def _arr(vals):
    return (ctypes.c_int * max(1, len(vals)))(*vals)


def _ws(lib, sizes, tile=(256, 256), max_pass=0, n=None):
    return lib.wn_backward_ragged_tiled_workspace_bytes(_arr([h for h, _ in sizes]), _arr([w for _, w in sizes]),
                                                        len(sizes) if n is None else n, tile[0], tile[1], max_pass)


def _table(n, windows):
    a256 = lambda v: (v + 255) // 256 * 256  # noqa: E731
    return a256(n * PACK_IN_ARGS_BYTES) + a256(n * RAGGED_GRADS_BYTES) + a256(windows * 72)


def test_header_declares_and_library_exports_the_new_entry_points(lib):
    header = open(os.path.join(ROOT, "include", "waternet_b200.h")).read()
    from waternet_b200 import _lib
    for name in NEW:
        assert f" {name}(" in header, name
        assert name in _lib.EXPORTED_SYMBOLS
        assert getattr(lib, name) is not None


def test_workspace_is_one_pass_plus_the_scratch_gradients_plus_the_table(lib):
    from waternet_b200.engine import ragged_plan
    # what does not depend on the pass: a 1 x 1 image alone is one pass of one pixel, one image and one window
    fixed = lib.wn_backward_tiled_workspace_bytes(1, 1, 1, 1, 1, 0) - TRAIN_BYTES_PER_PIXEL
    rng = random.Random(3)
    for tile, max_pass in [((256, 256), 0), ((998, 998), 0), ((20, 33), 50_000), ((1000, 1000), 1 << 20)]:
        sizes = [(rng.randint(1, 1500), rng.randint(1, 2000)) for _ in range(25)] + [(1, 1), (8, 24)]
        passes = ragged_plan(sizes, *tile, max_pass or DEFAULT_PASS)
        px = max(len(p["windows"]) * p["slot"][0] * p["slot"][1] for p in passes)
        windows = sum(len(p["windows"]) for p in passes)
        assert _ws(lib, sizes, tile, max_pass) == px * TRAIN_BYTES_PER_PIXEL + fixed + _table(len(sizes), windows)


def test_workspace_of_one_size_is_that_of_the_windowed_backward_plus_the_table(lib):
    from waternet_b200.engine import tile_geometry
    for n, h, w, tile, max_pass in [(3, 90, 130, (40, 40), 20_000), (2, 1080, 1920, (998, 998), 0), (5, 37, 53, (16, 8), 0)]:
        g = tile_geometry(h, w, *tile)
        got = _ws(lib, [(h, w)] * n, tile, max_pass)
        assert got == lib.wn_backward_tiled_workspace_bytes(n, h, w, *tile, max_pass) + _table(n, n * g["ny"] * g["nx"])


def test_workspace_does_not_grow_with_the_image_size_or_count(lib):
    from waternet_b200.engine import ragged_plan
    bound = DEFAULT_PASS * TRAIN_BYTES_PER_PIXEL + (64 << 20)  # dense and partial sums, parameter gradients
    for sizes in [[(3000, 4000)], [(3000, 4000)] * 8, [(1080, 1920)] * 40 + [(64, 64)] * 200, [(6000, 8000)] * 2]:
        windows = sum(len(p["windows"]) for p in ragged_plan(sizes, 998, 998, DEFAULT_PASS))
        assert _ws(lib, sizes, (998, 998)) - _table(len(sizes), windows) <= bound, sizes


def test_workspace_is_zero_for_rejected_arguments(lib):
    ok = [(37, 53), (1080, 1920)]
    assert _ws(lib, ok) > 0
    assert _ws(lib, ok, max_pass=TRAIN_MAX) > 0
    assert _ws(lib, ok, max_pass=TRAIN_MAX + 1) == 0                     # max_pass_pixels over 8 Mi
    assert _ws(lib, ok, max_pass=-1) == 0
    assert _ws(lib, [(2048, 4096)], tile=(2048, 4096)) > 0              # a window of exactly 8 Mi pixels
    assert _ws(lib, [(2048, 4097)], tile=(2048, 4097)) == 0              # a window over 8 Mi pixels
    assert _ws(lib, ok + [(3000, 3000)], tile=(3000, 3000)) == 0         # ... of one image of the list
    assert _ws(lib, ok, n=-1) == 0 and _ws(lib, [], n=0) == 0
    assert _ws(lib, [(1, 1)] * 65536, tile=(1, 1)) == 0                  # n over 65535
    assert _ws(lib, [(0, 5)]) == 0 and _ws(lib, [(5, -1)]) == 0
    assert _ws(lib, ok, tile=(0, 256)) == 0
    assert _ws(lib, [(30000, 30000)]) == 0                               # over the per-image size limit
    assert lib.wn_backward_ragged_tiled_workspace_bytes(None, _arr([5]), 1, 8, 8, 0) == 0
    assert lib.wn_backward_ragged_tiled_workspace_bytes(_arr([5]), None, 1, 8, 8, 0) == 0


def test_null_arguments_fail_with_a_message(lib):
    rc = lib.wn_backward_ragged_tiled(None, None, None, None, None, 1, 8, 8, 0, None, 0, None)
    assert rc == -1 and b"null argument" in lib.wn_last_error()


@pytest.mark.parametrize("seed", range(6))
def test_every_image_keeps_its_windows_contiguous_and_ascending(seed):
    """The fold's precondition: in plan order, the windows of one image form one run in ascending tile order."""
    from waternet_b200.engine import ragged_plan, tile_geometry
    rng = random.Random(seed)
    tile = (rng.randint(1, 300), rng.randint(1, 300))
    sizes = [(rng.randint(1, 700), rng.randint(1, 900)) for _ in range(rng.randint(1, 60))]
    max_pass = rng.choice([0, 10_000, 300_000, DEFAULT_PASS])
    order = [(r["img"], (r["rows"][0], r["cols"][0])) for p in ragged_plan(sizes, *tile, max_pass or DEFAULT_PASS)
             for r in p["windows"]]
    runs = {}
    for k, (img, _) in enumerate(order):
        runs.setdefault(img, []).append(k)
    assert sorted(runs) == list(range(len(sizes)))
    for img, pos in runs.items():
        g = tile_geometry(*sizes[img], *tile)
        assert len(pos) == g["ny"] * g["nx"]
        assert pos == list(range(pos[0], pos[0] + len(pos))), f"image {img} is not contiguous"
        kept = [order[k][1] for k in pos]
        assert kept == sorted(kept) and len(set(kept)) == len(kept), f"image {img} is not in tile order"
