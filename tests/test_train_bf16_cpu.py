"""The single-pass bf16 training arithmetic (WN_MODE_BF16) without a GPU: its replay bars, and the C ABI of its setter.

bf16_replay.emulate_* restate the kernels of that mode with exact float64 products: one bf16 product a_hi x w_hi per
product, fp32 results, every stored plane bf16(v) with lo = 0.  On every weight set and input kind their buffers and
parameter gradients must pass the replay bars (bf16_replay.check against the replay on the emulation's own decoded
buffers) and the exact-arithmetic bars (unrounded weights, 2^-8 M more); else a tau was fitted to luck.  Each fault
of bf16_replay.FAULTS -- an a_lo or w_lo pass left in, a lo plane not zeroed, g_lo x a_hi left in a weight gradient --
must fail the replay bar of the launch it targets.
"""
import ctypes
import os
import re

import pytest
import torch

import backward_reference as br
import bf16_replay as rp
import forward_reference as fr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPE = (1, 19, 24)
# forward launches (forward_reference numbering) -> the saved buffer that holds their output
FWD_BUFFER = {0: "a1", 1: "a2", 2: "a3", 3: "a4", 4: "a5", 5: "a6", 6: "a7", 7: "cm", 8: "r1", 9: "r2", 10: "refined"}


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(8, n))
    yield
    torch.set_num_threads(n)


def _grad(seed):
    return torch.randn(SHAPE[0], 3, *SHAPE[1:], generator=torch.Generator().manual_seed(seed))


def _vals(bufs):
    return {k: v.value for k, v in bufs.items()}


def _check_forward(sd, vals, tau_of=rp.launch_tau, exact=False, only=None):
    for layer, name in FWD_BUFFER.items():
        if only is not None and layer != only:
            continue
        src = vals["act0"] if layer in (0, 8) else vals[FWD_BUFFER[fr.INPUT_LAYER[layer]]]
        ref = rp.layer_replay(sd, layer, src, rounded=not exact)
        tau = tau_of(layer)
        rp.check(vals[name], ref, rp.exact_bar(tau) if exact else tau, f"forward {name}",
                 planes=name not in ("cm", "refined"))


def _check_backward(sd, stack, grad, vals, params, which=0, exact=False, only=None):
    for name, ref in rp.seed_replay(stack, grad, vals.get("cm"), vals.get("refined"), which).items():
        if only in (None, name):
            rp.check(vals[name], ref, rp.SEED_TAU, name, planes=True)
    for li in br.DGRAD:
        if li in vals and only in (None, li):
            mask = br.DGRAD_MASK[li]
            ref = rp.dgrad_replay(sd, li, vals[br.DGRAD_INPUT[li]], vals[mask] if mask else None, rounded=not exact)
            tau = rp.launch_tau(li)
            rp.check(vals[li], ref, rp.exact_bar(tau) if exact else tau, li, planes=True)
    for prefix, (dw, db) in params.items():
        if only not in (None, prefix):
            continue
        wref, bref = br.param_reference(prefix, vals)
        # the emulation sums exactly: the bar of the shortest partial sum
        rp.check(dw, wref, rp.wgrad_tau(0), f"{prefix}.weight")
        rp.check(db, bref, br.TAU["bias"], f"{prefix}.bias")


@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
@pytest.mark.parametrize("kind", fr.INPUT_KINDS)
def test_emulation_passes_the_replay_bars(weights, kind):
    sd = fr.weight_set(weights)
    ins = fr.make_inputs(kind, *SHAPE, seed=3)
    bufs = rp.emulate_forward(sd, ins)
    vals = _vals(bufs)
    _check_forward(sd, vals)
    for stack, which in (("all", 0), ("cmg", 0), ("refiner", 1)):
        out, params = rp.emulate_backward(sd, stack, _grad(7), bufs, which)
        _check_backward(sd, stack, _grad(7), _vals(out), params, which)


@pytest.mark.parametrize("weights", ("stress", "trained"))
def test_emulation_passes_the_exact_arithmetic_bars(weights):
    """Against the unrounded fp32 weights every launch stays within 2^-8 M + its accumulation bar."""
    sd = fr.weight_set(weights)
    bufs = rp.emulate_forward(sd, fr.make_inputs("floats", *SHAPE, seed=5))
    vals = _vals(bufs)
    _check_forward(sd, vals, exact=True)
    out, params = rp.emulate_backward(sd, "all", _grad(9), bufs)
    _check_backward(sd, "all", _grad(9), _vals(out), params, exact=True)


def test_bf16x3_results_fail_the_replay_bars():
    """The bars tell the modes apart: the bf16x3 emulation (three products, hi + lo planes) fails them."""
    sd = fr.weight_set("default")
    bufs = br.emulate_forward(sd, fr.make_inputs("floats", *SHAPE, seed=3))
    with pytest.raises(AssertionError):
        _check_forward(sd, _vals(bufs), only=3)


# (fault, where it is injected, the launch whose bar it must fail)
FAULT_CASES = [
    ("w_lo_pass", "forward", 3), ("a_lo_pass", "forward", 3), ("lo_not_zeroed", "forward", 3),
    ("w_lo_pass", "kD4", "kD4"), ("a_lo_pass", "kD4", "kD4"), ("lo_not_zeroed", "kD4", "kD4"),
    ("lo_not_zeroed", "g8", "g8"), ("g_lo_wgrad", "cmg.conv4", "cmg.conv4"),
    ("g_lo_wgrad", "wb_refiner.conv2", "wb_refiner.conv2"),
]


@pytest.mark.parametrize("fault,at,target", FAULT_CASES)
def test_each_fault_fails_its_launch(fault, at, target):
    sd = fr.weight_set("default")
    ins = fr.make_inputs("floats", *SHAPE, seed=3)
    grad = _grad(7)
    if at == "forward":
        bufs = rp.emulate_forward(sd, ins, fault, target)
        with pytest.raises(AssertionError):
            _check_forward(sd, _vals(bufs), only=target)
        return
    bufs = rp.emulate_forward(sd, ins)
    out, params = rp.emulate_backward(sd, "all", grad, bufs, fault=fault, fault_at=at)
    with pytest.raises(AssertionError):
        _check_backward(sd, "all", grad, _vals(out), params, only=target)


def test_set_train_mode_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "waternet_b200.h")).read()
    assert re.search(r"int\s+wn_set_train_mode\s*\(\s*wn_handle\s*\*\s*h\s*,\s*int\s+mode\s*\)\s*;", header)
    assert re.search(r"#define\s+WN_MODE_BF16\s+\(WN_MODE_BF16_FP8 \+ 1\)", header)  # = 3
    from waternet_b200 import _lib
    assert _lib.MODE_BF16 == 3
    lib = _lib.load()
    assert hasattr(lib, "wn_set_train_mode")
    version = int(re.search(r"#define\s+WN_ABI_VERSION\s+(\d+)", header).group(1))
    assert lib.wn_abi_version() == _lib.ABI_VERSION == version
    # a host-side setting: a NULL handle is refused without touching a device
    assert lib.wn_set_train_mode(None, _lib.MODE_BF16) == -1


def test_train_precision_attribute():
    from waternet_b200.net import TRAIN_PRECISIONS, WaterNet
    from waternet_b200 import _lib
    assert TRAIN_PRECISIONS == {"bf16x3": _lib.MODE_BF16X3, "bf16": _lib.MODE_BF16}
    m = WaterNet()
    assert m.train_precision == "bf16x3" and m._train_mode() == _lib.MODE_BF16X3
    m = WaterNet(train_precision="bf16")
    assert m._train_mode() == _lib.MODE_BF16 and m.cmg._train_mode() == _lib.MODE_BF16
    m.train_precision = "bf16x3"
    assert m.ce_refiner._train_mode() == _lib.MODE_BF16X3  # a bound stack follows its parent
    with pytest.raises(ValueError):
        WaterNet(train_precision="fp16")
    from waternet_b200.net import Refiner
    r = Refiner()
    r.train_precision = "bf16"
    assert r._train_mode() == _lib.MODE_BF16
    r.train_precision = "tf32"
    with pytest.raises(ValueError):
        r._train_mode()
