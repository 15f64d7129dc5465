"""Ragged batches of fp32 tensors without a GPU: the entry points of wn_forward_ragged and the ragged training step,
their workspace functions, the descriptor layout and the grouping of images into training calls."""
import ctypes
import os
import random

import pytest

from conftest import ROOT

BYTES_PER_PIXEL = 1868           # kUmmaBytesPerPixel: one pass of the tensor-core forward
TRAIN_MAX = 8 << 20              # pixels of one training pass
MODE_DEFAULT, MODE_FP32, MODE_BF16X3 = -1, 0, 1
NEW = ["wn_forward_ragged_workspace_bytes", "wn_forward_ragged", "wn_train_ragged_workspace_bytes",
       "wn_forward_train_ragged", "wn_backward_ragged"]


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def _arr(vals):
    return (ctypes.c_int * max(1, len(vals)))(*vals)


def _fwd_ws(lib, sizes, tile=(256, 256), max_pass=0, mode=MODE_DEFAULT):
    return lib.wn_forward_ragged_workspace_bytes(_arr([h for h, _ in sizes]), _arr([w for _, w in sizes]), len(sizes),
                                                 tile[0], tile[1], max_pass, mode)


def _train_ws(lib, sizes):
    return lib.wn_train_ragged_workspace_bytes(_arr([h for h, _ in sizes]), _arr([w for _, w in sizes]), len(sizes))


def test_header_declares_and_library_exports_the_new_entry_points(lib):
    header = open(os.path.join(ROOT, "include", "waternet_b200.h")).read()
    assert "#define WN_ABI_VERSION 11" in header
    assert "} wn_ragged_tensors;" in header
    from waternet_b200 import _lib
    for name in NEW:
        assert f" {name}(" in header, name
        assert name in _lib.EXPORTED_SYMBOLS
        assert getattr(lib, name) is not None
    assert lib.wn_abi_version() == 11


def test_descriptor_size_is_restated():
    from waternet_b200 import _lib
    assert ctypes.sizeof(_lib.RaggedTensors) == _lib.RAGGED_TENSORS_BYTES == 176
    assert _lib.RaggedTensors.in_strides.offset == 32 and _lib.RaggedTensors.out.offset == 160


def test_forward_workspace_is_the_largest_pass_plus_the_table(lib):
    from waternet_b200.engine import RAGGED_WINDOW_BYTES, ragged_plan
    a256 = lambda v: (v + 255) // 256 * 256  # noqa: E731
    rng = random.Random(5)
    for tile, max_pass in [((256, 256), 0), ((998, 998), 0), ((128, 96), 300_000)]:
        sizes = [(rng.randint(1, 1500), rng.randint(1, 2000)) for _ in range(30)]
        passes = ragged_plan(sizes, *tile, max_pass)
        px = max(len(p["windows"]) * p["slot"][0] * p["slot"][1] for p in passes)
        windows = sum(len(p["windows"]) for p in passes)
        table = a256(a256(len(sizes) * 160) + windows * RAGGED_WINDOW_BYTES)  # PackInArgs per image, then windows
        assert _fwd_ws(lib, sizes, tile, max_pass) == px * BYTES_PER_PIXEL + 4096 + 256 + table + 1024


def test_forward_workspace_is_zero_for_rejected_arguments(lib):
    ok = [(37, 53), (1080, 1920)]
    assert _fwd_ws(lib, ok) > 0 and _fwd_ws(lib, ok, mode=MODE_BF16X3) > 0
    assert _fwd_ws(lib, ok, mode=MODE_FP32) == 0                  # WN_E_UNSUPPORTED
    assert _fwd_ws(lib, ok, mode=7) == 0
    assert _fwd_ws(lib, []) == 0
    assert _fwd_ws(lib, [(0, 5)]) == 0 and _fwd_ws(lib, [(5, -1)]) == 0
    assert _fwd_ws(lib, ok, tile=(0, 256)) == 0
    assert _fwd_ws(lib, ok, max_pass=-1) == 0
    assert _fwd_ws(lib, [(30000, 30000)]) == 0                     # over the per-image size limit
    assert lib.wn_forward_ragged_workspace_bytes(None, _arr([5]), 1, 8, 8, 0, -1) == 0


def test_train_workspace_is_zero_for_rejected_arguments(lib):
    assert _train_ws(lib, [(37, 53), (113, 117)]) > 0
    assert _train_ws(lib, []) == 0
    assert _train_ws(lib, [(0, 4)]) == 0 and _train_ws(lib, [(4, -2)]) == 0
    assert _train_ws(lib, [(2048, 4096)]) > 0                       # exactly 8 Mi pixels
    assert _train_ws(lib, [(2048, 4097)]) == 0
    assert _train_ws(lib, [(2048, 2048), (1, 2049)]) == 0           # the slot is the per-axis maximum: 2 x 2048 x 2049
    assert _train_ws(lib, [(1, 1)] * 65535) > 0
    assert _train_ws(lib, [(1, 1)] * 65536) == 0
    assert lib.wn_train_ragged_workspace_bytes(None, _arr([5]), 1) == 0


def test_train_workspace_grows_with_the_slot_not_the_images(lib):
    a = _train_ws(lib, [(100, 40), (40, 100)])
    b = _train_ws(lib, [(100, 100), (100, 100)])
    assert a == b  # two 100 x 100 slots either way
    per_px = (_train_ws(lib, [(100, 100)] * 3) - b)
    assert 5000 < per_px / 10_000 < 6000  # ~5.6 KB per slot pixel


@pytest.mark.parametrize("seed", range(4))
def test_training_calls_keep_the_c_limits(lib, seed):
    from waternet_b200.engine import ragged_train_calls
    rng = random.Random(seed)
    sizes = [(rng.randint(1, 600), rng.randint(1, 800)) for _ in range(400)] + [(2048, 4096), (1, 1), (1, 8000)]
    calls = ragged_train_calls(sizes, TRAIN_MAX)
    assert sorted(i for c in calls for i in c) == list(range(len(sizes)))
    for c in calls:
        sub = [sizes[i] for i in c]
        sh, sw = max(h for h, _ in sub), max(w for _, w in sub)
        assert len(c) * sh * sw <= TRAIN_MAX and len(c) <= 65535
        if len(c) > 1:
            assert 4 * (len(c) * sh * sw - sum(h * w for h, w in sub)) <= len(c) * sh * sw
        assert _train_ws(lib, sub) > 0  # every call is one the library accepts
    # a lower limit only splits further
    assert len(ragged_train_calls(sizes, 1 << 20)) >= len(calls)


def test_training_calls_of_equal_sizes_fill_the_pass():
    from waternet_b200.engine import ragged_train_calls
    calls = ragged_train_calls([(112, 112)] * 1000, TRAIN_MAX)
    assert [len(c) for c in calls] == [668, 332]  # 668 x 112 x 112 <= 8 Mi < 669 x 112 x 112
    assert calls[0] == list(range(668))
