"""Without a GPU: the float64 restatement of d(1 - SSIM)/d(out) against torch autograd, the GPU bar against mutations
of the restatement, the refusals of ssim_loss and wn_ssim_grad, the exported symbols, and --ssim-weight."""
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
import ssim_grad_reference as sgr
from conftest import ROOT
from waternet_b200 import _lib
from waternet_b200 import training as T
from waternet_b200.metrics import ssim, ssim_loss

SIZES = [(6, 6), (8, 40), (10, 10), (11, 11), (12, 13), (64, 97)]
# torch's float64 moments of nearly constant values (E[x^2] ~ 0.25 against variances ~1e-7) cancel: its own
# error is ~2.5e6 x 2^-53 per moment, so on "flat" the two agree to that, not to 1e-12
REL = {"noise": 1e-12, "smooth": 1e-12, "flat": 1e-7}


def torch_grad(out, ref, dtype=torch.float64):
    """torch autograd of 1 - ssim (a batch) or 1 - batch_quality(...)[0] (lists), as numpy."""
    if isinstance(out, (list, tuple)):
        to = [torch.from_numpy(o).to(dtype).requires_grad_() for o in out]
        s = T.batch_quality(to, [torch.from_numpy(r).to(dtype) for r in ref])[0]
        return [g.double().numpy() for g in torch.autograd.grad(1 - s, to)]
    to = torch.from_numpy(out).to(dtype).requires_grad_()
    return torch.autograd.grad(1 - ssim(to, torch.from_numpy(ref).to(dtype)), to)[0].double().numpy()


def _rel(got, want):
    if isinstance(got, list):
        return max(np.abs(g - w).max() for g, w in zip(got, want)) / max(np.abs(w).max() for w in want)
    return np.abs(got - want).max() / np.abs(want).max()


@pytest.mark.parametrize("kind", ["noise", "smooth", "flat"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_restatement_matches_torch_autograd_in_float64(size, kind):
    for n in (1, 2, 3):
        o, r = mref.inputs(kind, (n, 3, *size), seed=size[0] + n)
        assert _rel(sgr.grad(o, r), torch_grad(o, r)) <= REL[kind], (size, n)


@pytest.mark.parametrize("kind", ["noise", "smooth"])
def test_restatement_matches_torch_autograd_for_a_list(kind):
    pairs = [mref.inputs(kind, (1 + k % 3, 3, *s), seed=k) for k, s in enumerate(SIZES)]
    o, r = [a for a, _ in pairs], [b for _, b in pairs]
    assert _rel(sgr.grad(o, r), torch_grad(o, r)) <= REL[kind]


def tied(shape, seed=0):
    """out with many elements at its max (1) and min (0), as a ReLU and a clamp leave them; ref inside (0.1, 0.9)."""
    rng = np.random.default_rng(seed)
    o = np.clip(1.4 * rng.random(shape) - 0.2, 0, 1).astype(np.float32)
    r = (0.1 + 0.8 * rng.random(shape)).astype(np.float32)
    return o, r


def equal_ranges(shape, seed=0):
    """out and ref both with min 0 and max 1: torch.maximum splits the range's gradient half and half."""
    rng = np.random.default_rng(seed)
    o, r = rng.random(shape).astype(np.float32), rng.random(shape).astype(np.float32)
    for a in (o, r):
        a.reshape(-1)[:2] = (0.0, 1.0)
    return o, r


def ref_larger(shape, seed=0):
    """ref's range larger than out's: no range gradient reaches out."""
    rng = np.random.default_rng(seed)
    o = (0.3 + 0.4 * rng.random(shape)).astype(np.float32)
    return o, rng.random(shape).astype(np.float32)


@pytest.mark.parametrize("make", [tied, equal_ranges, ref_larger])
@pytest.mark.parametrize("size", [(8, 40), (12, 13), (64, 97)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_restatement_range_rules_match_torch(make, size):
    o, r = make((2, 3, *size))
    if make is tied:
        assert (o == 1).sum() > 10 and (o == 0).sum() > 10
    assert _rel(sgr.grad(o, r), torch_grad(o, r)) <= 1e-12
    lo, lr = [o[:1], o[1:]], [r[:1], r[1:]]
    assert _rel(sgr.grad(lo, lr), torch_grad(lo, lr)) <= 1e-12


def test_ref_range_larger_sends_nothing_to_the_extremes():
    o, r = ref_larger((1, 3, 20, 30))
    with_range = sgr.grad(o, r)
    assert np.array_equal(with_range, sgr.grad(o, r, range_term=False))


def _violations(o, r, **mutation):
    want, m = sgr.grad(o, r, terms=True)
    t32 = torch_grad(o, r, torch.float32)
    assert sgr.bar_violations(want, want, t32, m)[0] == 0
    return sgr.bar_violations(sgr.grad(o, r, **mutation), want, t32, m)


@pytest.mark.parametrize("case", ["range_term", "split_ties", "fold", "crop", "pool_items"])
def test_the_bar_rejects_each_mutation(case):
    """Each broken rule moves d(out) beyond 4 max(torch fp32's worst error, F) somewhere."""
    if case == "range_term":
        r, o = mref.inputs("noise", (2, 3, 40, 50), seed=1)  # out the clipped one: its range is the larger
        bad = _violations(o, r, range_term=False)
    elif case == "split_ties":
        o, r = tied((2, 3, 40, 50))
        bad = _violations(o, r, split_ties=False)
    elif case == "fold":
        o, r = mref.inputs("noise", (2, 3, 8, 40), seed=2)
        bad = _violations(o, r, fold=False)
    elif case == "crop":
        o, r = mref.inputs("noise", (2, 3, 64, 97), seed=3)
        bad = _violations(o, r, crop=False)
    else:
        pairs = [mref.inputs("noise", (1 + k, 3, 24, 30), seed=k) for k in range(3)]
        bad = _violations([a for a, _ in pairs], [b for _, b in pairs], pool_items=True)
    assert bad[0] > 0, bad


def test_sides_of_five_or_less_and_bad_shapes_are_refused():
    for shape in [(1, 3, 5, 9), (1, 3, 9, 5)]:
        a = torch.rand(shape)
        with pytest.raises(ValueError, match="padding"):
            ssim_loss(a, a)
        with pytest.raises(ValueError, match="padding"):
            ssim_loss([torch.rand(1, 3, 8, 8), a], [torch.rand(1, 3, 8, 8), a])
    with pytest.raises(ValueError, match="shape"):
        ssim_loss(torch.rand(1, 3, 8, 8), torch.rand(1, 3, 8, 9))
    with pytest.raises(ValueError, match="shape"):
        ssim_loss(torch.rand(1, 4, 8, 8), torch.rand(1, 4, 8, 8))
    with pytest.raises(ValueError, match="lists"):
        ssim_loss([torch.rand(1, 3, 8, 8)], [])


def test_cpu_tensors_are_refused_there_is_no_cpu_path():
    a = torch.rand(2, 3, 16, 16, requires_grad=True)
    with pytest.raises(_lib.WaterNetLibraryError):
        ssim_loss(a, a.detach())
    with torch.no_grad(), pytest.raises(_lib.WaterNetLibraryError):
        ssim_loss(a, a)


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import build
    build.build()
    return _lib.load()


def test_new_symbols_are_declared_and_exported(lib):
    """include/waternet_b200_ssim.h declares exactly SSIM_SYMBOLS, the library exports them, neither existing header
    mentions them, and the ABI version is still 11."""
    text = re.sub(r"/\*.*?\*/", "", open(f"{ROOT}/include/waternet_b200_ssim.h").read(), flags=re.S)
    declared = sorted(set(re.findall(r"\b(wn_[a-z0-9_]+)\s*\(", text)))
    assert declared == sorted(_lib.SSIM_SYMBOLS) == ["wn_ssim_grad", "wn_ssim_grad_workspace_bytes"]
    assert all(hasattr(lib, name) for name in declared)
    assert not set(declared) & (set(_lib.EXPORTED_SYMBOLS) | set(_lib.METRICS_SYMBOLS))
    for header in ("waternet_b200.h", "waternet_b200_metrics.h"):
        assert "wn_ssim" not in open(f"{ROOT}/include/{header}").read(), header
    assert lib.wn_abi_version() == _lib.ABI_VERSION == 11
    assert ctypes.sizeof(_lib.SSIMGradImage) == 48


def _sizes(sizes):
    return (ctypes.c_int * len(sizes))(*[h for h, _ in sizes]), (ctypes.c_int * len(sizes))(*[w for _, w in sizes])


def test_workspace_is_zero_for_rejected_sizes_and_small_per_pixel(lib):
    ws = lambda sizes: lib.wn_ssim_grad_workspace_bytes(*_sizes(sizes), len(sizes))  # noqa: E731
    assert ws([(6, 6)]) > 0 and ws([(5, 6)]) == 0 and ws([(6, 5)]) == 0 and ws([(6, 0)]) == 0
    assert ws([(16, 0x7fffffff // 3 // 16 + 1)]) == 0
    assert lib.wn_ssim_grad_workspace_bytes(*_sizes([(8, 8)]), 0) == 0
    assert lib.wn_ssim_grad_workspace_bytes(None, None, 1) == 0
    big = ws([(1080, 1920)] * 4)
    assert lib.wn_quality_workspace_bytes(*_sizes([(1080, 1920)] * 4), 4) < big < 4 * 1080 * 1920 * 160 / 1024, big  # ~140 bytes per 1024 pixels


def test_call_refusals_before_any_device_work(lib):
    """With a stand-in handle (a zero-filled host buffer) and fake, disjoint device addresses: every refusal returns
    its code before the call touches the device or counts a launch."""
    handle = ctypes.create_string_buffer(64 * 1024)
    h = ctypes.addressof(handle)
    base = 0x10000000

    def call(sizes, groups, scales=None, grads=None, stats=base, ws_bytes=1 << 40, n=None, table=True):
        t = (_lib.SSIMGradImage * max(1, len(sizes)))()
        for i, (d, (hh, ww), g) in enumerate(zip(t, sizes, groups)):
            d.out, d.ref, d.grad = base + (3 * i + 1) * (1 << 24), base + (3 * i + 2) * (1 << 24), \
                base + (3 * i + 3) * (1 << 24)
            if grads is not None and grads[i] is not None:
                d.grad = grads[i]
            d.height, d.width, d.group, d.scale = hh, ww, g, 1.0 if scales is None else scales[i]
        rc = lib.wn_ssim_grad(h, t if table else None, len(sizes) if n is None else n, stats, base, ws_bytes, None)
        return rc, lib.wn_last_error().decode()

    assert lib.wn_ssim_grad(None, None, 1, base, base, 1, None) == -1
    assert call([(8, 8)], [0], table=False)[0] == -1
    assert call([(8, 8)], [0], stats=None)[0] == -1
    assert call([(8, 8)], [0], grads=[0]) == (-1, "wn_ssim_grad: null image pointer (image 0)")
    assert call([(8, 8)], [0], n=0) == (-1, "wn_ssim_grad: 1..65535 images per call, got n=0")
    assert call([(8, 8)], [0], n=65536)[0] == -5
    assert call([(8, 8), (8, 8)], [0, 2]) == (-1, "wn_ssim_grad: image 1: group 2 outside 0..1")
    assert call([(8, 8)], [-1])[0] == -1
    for bad in (float("nan"), float("inf"), -float("inf")):
        rc, msg = call([(8, 8), (8, 8)], [0, 1], scales=[1.0, bad])
        assert rc == -1 and "image 1: scale" in msg and "not finite" in msg, msg
    out0 = base + 1 * (1 << 24)
    for g in (out0, out0 + 4 * 3 * 8 * 8 - 4, base + 5 * (1 << 24) + 100, base + 6 * (1 << 24) - 8):
        rc, msg = call([(8, 8), (8, 8)], [0, 1], grads=[g, None])  # onto out 0, its end, ref 1, below grad 1
        assert rc == -1 and "overlaps" in msg, (hex(g), msg)
    rc, msg = call([(8, 8), (5, 8)], [0, 1])
    assert rc == -1 and "image 1 is 5 x 8" in msg and "at least 6" in msg
    assert call([(8, 8), (0, 8)], [0, 0])[0] == -1
    assert call([(16, 0x7fffffff // 3 // 16 + 1)], [0])[0] == -5
    assert call([(8, 8)], [0], stats=base + 4) == (-1, "wn_ssim_grad: stats is not 8-byte aligned")
    need = lib.wn_ssim_grad_workspace_bytes(*_sizes([(8, 8)]), 1)
    assert call([(8, 8)], [0], ws_bytes=need - 1) == (-4, "wn_ssim_grad: workspace too small")
    assert lib.wn_launch_count(h) == 0


def test_ssim_weight_is_parsed_refused_when_negative_and_recorded(tmp_path):
    ap = argparse.ArgumentParser()
    T.add_loss_arg(ap)
    assert T.loss_config(ap.parse_args([])) == {"ssim_weight": 0.0}
    args = ap.parse_args(["--ssim-weight", "0.5"])
    T.save_metrics(tmp_path, None, None, {"epochs": 1, **T.loss_config(args)})
    assert json.loads((tmp_path / "config.json").read_text())["ssim_weight"] == 0.5
    for bad in ("-0.1", "nan", "inf", "x"):
        with pytest.raises(SystemExit):
            ap.parse_args(["--ssim-weight", bad])
    src = open(f"{ROOT}/train.py").read()
    assert "T.add_loss_arg(ap)" in src and "**T.loss_config(args)" in src and "ssim_weight=args.ssim_weight" in src


def test_train_py_refuses_a_negative_ssim_weight():
    res = subprocess.run([sys.executable, "train.py", "--ssim-weight", "-1"], cwd=ROOT, capture_output=True,
                         text=True, timeout=300)
    assert res.returncode == 2 and "--ssim-weight" in res.stderr and "at least 0" in res.stderr, res.stderr
