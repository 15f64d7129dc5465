"""Without a GPU: the float64 restatement the native metrics are checked against, the refusals of native_quality,
wn_quality and --metrics, the exported symbols, and --metrics in config.json."""
import argparse
import ctypes
import json
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import metrics_reference as mref
from conftest import ROOT
from waternet_b200 import _lib
from waternet_b200 import training as T
from waternet_b200.metrics import native_quality, psnr, ssim

SIZES = [(6, 6), (11, 11), (12, 13), (64, 97), (112, 112)]


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import build
    build.build()
    return _lib.load()


@pytest.mark.parametrize("kind", ["noise", "smooth"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_restatement_matches_metrics_in_float64_for_a_batch(size, kind):
    o, r = mref.inputs(kind, (3, 3, *size), seed=size[0])
    to, tr = torch.from_numpy(o).double(), torch.from_numpy(r).double()
    s, p = mref.quality(o, r)
    assert abs(s - ssim(to, tr).item()) <= 1e-12
    assert abs(p - psnr(to, tr, 1.0).item()) <= 1e-12


@pytest.mark.parametrize("kind", ["noise", "smooth"])
def test_restatement_matches_batch_quality_in_float64_for_a_list(kind):
    pairs = [mref.inputs(kind, (1 + k % 2, 3, *size), seed=k) for k, size in enumerate(SIZES)]
    outs, refs = [o for o, _ in pairs], [r for _, r in pairs]
    s, p = mref.quality(outs, refs)
    ts, tp = T.batch_quality([torch.from_numpy(o).double() for o in outs], [torch.from_numpy(r).double() for r in refs])
    assert abs(s - ts.item()) <= 1e-12
    assert abs(p - tp.item()) <= 1e-12


def test_restatement_of_a_constant_pair_is_nan_like_torch():
    o = np.full((1, 3, 12, 12), 0.25, np.float32)
    assert np.isnan(mref.quality(o, o)[0]) and torch.isnan(ssim(torch.from_numpy(o), torch.from_numpy(o)))


@pytest.mark.parametrize("shape", [(1, 3, 5, 9), (1, 3, 9, 5), (2, 3, 1, 1)])
def test_sides_of_five_or_less_are_refused_like_torch(shape):
    a = torch.rand(shape)
    with pytest.raises(RuntimeError, match="Padding size"):
        ssim(a, a)
    with pytest.raises(ValueError, match="padding"):
        native_quality(a, a)
    with pytest.raises(ValueError, match="padding"):
        native_quality([torch.rand(1, 3, 8, 8), a], [torch.rand(1, 3, 8, 8), a])


def test_shape_mismatch_and_bad_lists_are_refused():
    with pytest.raises(ValueError, match="shape"):
        native_quality(torch.rand(1, 3, 8, 8), torch.rand(1, 3, 8, 9))
    with pytest.raises(ValueError, match="shape"):
        native_quality(torch.rand(1, 4, 8, 8), torch.rand(1, 4, 8, 8))
    with pytest.raises(ValueError, match="lists"):
        native_quality([torch.rand(1, 3, 8, 8)], [])
    with pytest.raises(ValueError, match="lists"):
        native_quality([], [])


def test_cpu_tensors_are_refused_there_is_no_cpu_path():
    a = torch.rand(2, 3, 16, 16)
    with pytest.raises(_lib.WaterNetLibraryError):
        native_quality(a, a)
    with pytest.raises(_lib.WaterNetLibraryError):
        T.batch_quality(a, a, native=True)


@pytest.mark.parametrize("script", ["train.py", "score.py"])
def test_unknown_metrics_value_is_refused(script):
    res = subprocess.run([sys.executable, script, "--weights", "w.pt", "--metrics", "fast"], cwd=ROOT,
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 2 and "invalid choice: 'fast'" in res.stderr, res.stderr


def test_metrics_setting_is_recorded_in_config_json(tmp_path):
    ap = argparse.ArgumentParser()
    T.add_metrics_arg(ap)
    assert T.metrics_config(ap.parse_args([])) == {"metrics": "torch"}
    args = ap.parse_args(["--metrics", "native"])
    T.save_metrics(tmp_path, None, None, {"epochs": 1, **T.metrics_config(args)})
    assert json.loads((tmp_path / "config.json").read_text())["metrics"] == "native"
    src = open(f"{ROOT}/train.py").read()
    assert "T.add_metrics_arg(ap)" in src and "**T.metrics_config(args)" in src


def test_new_symbols_are_declared_and_exported(lib):
    """include/waternet_b200_metrics.h declares what the binding's METRICS_SYMBOLS names, the library exports it,
    and the enhancement header declares none of it."""
    text = re.sub(r"/\*.*?\*/", "", open(f"{ROOT}/include/waternet_b200_metrics.h").read(), flags=re.S)
    declared = sorted(set(re.findall(r"\b(wn_[a-z0-9_]+)\s*\(", text)))
    assert declared == sorted(_lib.METRICS_SYMBOLS) == ["wn_quality", "wn_quality_workspace_bytes"]
    assert all(hasattr(lib, name) for name in declared)
    assert not set(declared) & set(_lib.EXPORTED_SYMBOLS)
    assert "wn_quality" not in open(f"{ROOT}/include/waternet_b200.h").read()
    assert "#define WN_QUALITY_STATS 7" in text and _lib.QUALITY_STATS == 7
    assert ctypes.sizeof(_lib.QualityImage) == 32


def _sizes(sizes):
    return (ctypes.c_int * len(sizes))(*[h for h, _ in sizes]), (ctypes.c_int * len(sizes))(*[w for _, w in sizes])


def test_workspace_is_zero_for_rejected_sizes_and_small_per_pixel(lib):
    ws = lambda sizes: lib.wn_quality_workspace_bytes(*_sizes(sizes), len(sizes))  # noqa: E731
    assert ws([(6, 6)]) > 0 and ws([(5, 6)]) == 0 and ws([(6, 5)]) == 0 and ws([(6, 0)]) == 0
    assert ws([(16, 0x7fffffff // 3 // 16 + 1)]) == 0
    assert lib.wn_quality_workspace_bytes(*_sizes([(8, 8)]), 0) == 0
    assert lib.wn_quality_workspace_bytes(None, None, 1) == 0
    big = ws([(1080, 1920)] * 4)
    assert big < 4 * 1080 * 1920 * 48 / 1024, big  # ~40 bytes per 1024 pixels


def test_call_refusals_before_any_device_work(lib):
    """With a stand-in handle (a zero-filled host buffer) and fake device addresses: every refusal returns before
    the call touches the device."""
    handle = ctypes.create_string_buffer(64 * 1024)
    h = ctypes.addressof(handle)
    fake = 0x10000

    def call(sizes, groups, stats=fake, ws_bytes=1 << 40, n=None, table=True):
        t = (_lib.QualityImage * max(1, len(sizes)))()
        for d, (hh, ww), g in zip(t, sizes, groups):
            d.out, d.ref, d.height, d.width, d.group = fake, fake, hh, ww, g
        rc = lib.wn_quality(h, t if table else None, len(sizes) if n is None else n, stats, fake, ws_bytes, None)
        return rc, lib.wn_last_error().decode()

    assert lib.wn_quality(None, None, 1, fake, fake, 1, None) == -1
    assert call([(8, 8)], [0], table=False)[0] == -1
    assert call([(8, 8)], [0], stats=None)[0] == -1
    assert call([(8, 8)], [0], n=0) == (-1, "wn_quality: 1..65535 images per call, got n=0")
    assert call([(8, 8)], [0], n=65536)[0] == -5
    assert call([(8, 8), (8, 8)], [0, 2]) == (-1, "wn_quality: image 1: group 2 outside 0..1")
    assert call([(8, 8)], [-1])[0] == -1
    rc, msg = call([(8, 8), (5, 8)], [0, 1])
    assert rc == -1 and "image 1 is 5 x 8" in msg and "at least 6" in msg
    assert call([(8, 8), (0, 8)], [0, 0])[0] == -1
    assert call([(16, 0x7fffffff // 3 // 16 + 1)], [0])[0] == -5
    assert call([(8, 8)], [0], stats=fake + 4) == (-1, "wn_quality: stats is not 8-byte aligned")
    need = lib.wn_quality_workspace_bytes(*_sizes([(8, 8)]), 1)
    assert call([(8, 8)], [0], ws_bytes=need - 1) == (-4, "wn_quality: workspace too small")
