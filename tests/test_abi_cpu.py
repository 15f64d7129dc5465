"""CPU-side checks: the C-ABI library loads and exports what include/*.h declares; host logic."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import forward as ofw
from oracle import preprocess as opre


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "waternet_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(wn_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(lib):
    from waternet_b200 import _lib
    declared = _declared_symbols()
    assert len(declared) >= 12
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/waternet_b200.h but not exported"
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared, "ctypes binding and header disagree"
    assert lib.wn_abi_version() == _lib.ABI_VERSION == int(
        re.search(r"#define\s+WN_ABI_VERSION\s+(\d+)", open(os.path.join(ROOT, "include", "waternet_b200.h")).read()).group(1))


def test_constant_tables_match_oracle(lib):
    gtab = (ctypes.c_uint16 * 256)()
    ctab = (ctypes.c_uint16 * 3072)()
    ytab = (ctypes.c_int16 * 256)()
    fytab = (ctypes.c_int16 * 256)()
    igtab = (ctypes.c_uint8 * 4096)()
    gamma = (ctypes.c_uint8 * 256)()
    div255 = (ctypes.c_float * 256)()
    assert lib.wn_build_tables_host(gtab, ctab, ytab, fytab, igtab, gamma, div255) == 0
    assert np.array_equal(np.array(gtab), opre._GTAB)
    assert np.array_equal(np.array(ctab), opre._CTAB)
    assert np.array_equal(np.array(ytab), opre._YTAB)
    assert np.array_equal(np.array(fytab), opre._FYTAB)
    assert np.array_equal(np.array(igtab), opre._IGTAB)
    levels = np.arange(256, dtype=np.uint8)
    assert np.array_equal(np.array(gamma), opre.gamma_correction(levels))
    assert np.array_equal(np.array(div255, dtype=np.float32), levels.astype(np.float32) / np.float32(255))


def test_null_arguments_are_rejected_without_a_gpu(lib):
    assert lib.wn_create(0, None) != 0
    assert b"NULL" in lib.wn_last_error() or b"null" in lib.wn_last_error()
    assert lib.wn_forward_workspace_bytes(0, 10, 10, 0) == 0
    assert lib.wn_forward_workspace_bytes(2, 112, 112, 0) > 0
    assert lib.wn_preprocess_workspace_bytes(2, 112, 112) > 0
    assert lib.wn_submodule_workspace_bytes(2, 112, 112, -1) > lib.wn_forward_workspace_bytes(2, 112, 112, -1)
    assert lib.wn_enhance_workspace_bytes(2, 112, 112, -1) > 0
    assert lib.wn_train_workspace_bytes(65535, 1, 1) > 0
    assert lib.wn_train_workspace_bytes(65536, 1, 1) == 0   # at most 65535 images per training call
    assert lib.wn_train_workspace_bytes(0, 8, 8) == 0
    assert lib.wn_forward_chunk_images(None, 4, 8, 8) == 0 and lib.wn_f8_overflowed(None) == 0
    assert lib.wn_set_chunk_pixels(None, 0) != 0


def test_debug_layer_bound(lib):
    """wn_debug_forward_layer numbers the launch outputs 0..10 (10: the three refined images, Engine.LAYER_CHANNELS);
    the layer is checked before anything else, so the bound shows without a device."""
    from waternet_b200.engine import Engine
    assert Engine.LAYER_CHANNELS == (128, 128, 128, 64, 64, 64, 64, 3, 96, 96, 9)
    call = lambda layer: lib.wn_debug_forward_layer(None, None, None, None, None, None, 1, 1, 1, 0, layer, None, None,
                                                    0, None)
    for layer in (-1, 11):
        assert call(layer) != 0 and b"not in 0..10" in lib.wn_last_error()
    for layer in (0, 10):
        assert call(layer) != 0 and b"bad argument" in lib.wn_last_error()


def test_debug_backward_layer_bound(lib):
    """wn_debug_backward_layer numbers its buffers 0..24 (Engine.BACKWARD_BUFFER_CHANNELS, the header's table); the
    number is checked before anything else, then the stack, so both bounds show without a device."""
    from waternet_b200 import _lib
    from waternet_b200.engine import Engine
    assert len(Engine.BACKWARD_BUFFER_CHANNELS) == _lib.DEBUG_BACKWARD_BUFFERS == 25
    text = open(os.path.join(ROOT, "include", "waternet_b200.h")).read()
    assert int(re.search(r"#define\s+WN_DEBUG_BACKWARD_BUFFERS\s+(\d+)", text).group(1)) == 25
    call = lambda stack, which, buffer: lib.wn_debug_backward_layer(None, stack, which, buffer, None, None, 1, 1, 1,
                                                                    None, None, 0, None)
    for buffer in (-1, 25):
        assert call(-1, 0, buffer) != 0 and b"not in 0..24" in lib.wn_last_error()
    for stack, which in ((-2, 0), (2, 0), (1, -1), (1, 3)):
        assert call(stack, which, 0) != 0 and b"stack must be" in lib.wn_last_error()
    for stack, which, buffer in ((-1, 0, 0), (0, 0, 24), (1, 2, 13)):
        assert call(stack, which, buffer) != 0 and b"null argument" in lib.wn_last_error()


def test_state_dict_is_reference_compatible():
    from waternet_b200.net import WaterNet
    m = WaterNet()
    sd = m.state_dict()
    spec = ofw.state_dict_spec()
    assert list(sd.keys()) == [k for k, _ in spec]
    for k, shape in spec:
        assert tuple(sd[k].shape) == shape
    m.load_state_dict(ofw.synthetic_state_dict(0), strict=True)
    assert sum(p.numel() for p in m.parameters()) == 1_090_668
    ordered = m._ordered_params()
    assert len(ordered) == 34 and all(a is b for a, b in zip(ordered, m.parameters()))


def test_torch_graph_equals_oracle_on_cpu():
    """The differentiable graph used for gradients is the same function as the oracle."""
    from waternet_b200.net import WaterNet
    m = WaterNet()
    sd = ofw.synthetic_state_dict(1, 3.0)
    m.load_state_dict(sd)
    torch.manual_seed(0)
    ins = [torch.rand(1, 3, 20, 24) for _ in range(4)]
    with torch.no_grad():
        a = m._graph(*ins)
    b = ofw.waternet_forward(sd, *ins)
    assert torch.allclose(a, b, rtol=1e-5, atol=1e-6)


def test_no_cpu_fallback_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from waternet_b200 import WaterNetLibraryError, data
    from waternet_b200.hub import waternet
    with pytest.raises(WaterNetLibraryError):
        data.transform(ofw.synthetic_image(0, 16, 16))
    with pytest.raises(WaterNetLibraryError):
        waternet(pretrained=False)
    # the reference's waternet(device=None) hands back a CPU model (hubconf.py:96); this build is CUDA-only and
    # says so at the call instead of failing later (INTEGRATION.md "Differences")
    with pytest.raises(WaterNetLibraryError, match="CUDA"):
        waternet(pretrained=False, device=None)
    with pytest.raises(WaterNetLibraryError):
        waternet(pretrained=False, device="cpu")
    # sub-modules and the model refuse CPU tensors the same way
    from waternet_b200.net import ConfidenceMapGenerator, Refiner, WaterNet
    t = torch.rand(1, 3, 8, 8)
    with torch.no_grad():
        for call in (lambda: WaterNet()(t, t, t, t), lambda: ConfidenceMapGenerator()(t, t, t, t),
                     lambda: Refiner()(t, t)):
            with pytest.raises(WaterNetLibraryError):
                call()


def test_packed_weight_cache_key_tracks_parameter_changes():
    """Host logic of the packed-weight cache (advisor finding): the epoch advances on load_state_dict / .to() /
    invalidate_packed_weights(), _version on in-place updates; deepcopy and pickling keep the parent binding."""
    import copy
    import io
    from waternet_b200.net import WaterNet, _param_version
    m = WaterNet()
    e0 = getattr(m, "_pack_epoch", 0)
    m.load_state_dict(ofw.synthetic_state_dict(0))
    e1 = m._pack_epoch
    assert e1 > e0 and m.cmg._pack_epoch >= 1
    m.float()
    assert m._pack_epoch > e1
    v0 = _param_version(m.cmg.conv1.weight)
    with torch.no_grad():
        m.cmg.conv1.weight.mul_(2.0)
    assert _param_version(m.cmg.conv1.weight) > v0
    e2 = m._pack_epoch
    m.cmg.conv1.weight.data.mul_(0.5)      # invisible to _version: the documented manual hook
    m.invalidate_packed_weights()
    assert m._pack_epoch > e2
    twin = copy.deepcopy(m)
    assert twin.cmg._parent_ref() is twin and twin.gc_refiner._slot == 2 and m.cmg._parent_ref() is m
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert again.wb_refiner._parent_ref() is again
    with torch.inference_mode():
        p = torch.nn.Parameter(torch.zeros(1))
    assert isinstance(_param_version(p), int)


def test_submodules_are_the_reference_graph_when_autograd_records():
    """ConfidenceMapGenerator / Refiner are callable like the reference's (net.py:45-56, 75-80); with autograd
    recording they evaluate the torch graph (CPU works), which must be the oracle's function."""
    from waternet_b200.net import WaterNet
    m = WaterNet()
    sd = ofw.synthetic_state_dict(2, 3.0)
    m.load_state_dict(sd)
    torch.manual_seed(1)
    x, wb, he, gc = [torch.rand(1, 3, 12, 14) for _ in range(4)]
    maps = m.cmg(x, wb, he, gc)
    assert isinstance(maps, tuple) and len(maps) == 3 and maps[0].shape == (1, 1, 12, 14) and maps[0].requires_grad
    ref = ofw.confidence_maps(sd, x, wb, he, gc)
    assert torch.allclose(torch.cat(maps, 1), ref, rtol=1e-5, atol=1e-6)
    r = m.ce_refiner(x, he)
    assert torch.allclose(r, ofw.refine(sd, "ce_refiner", x, he), rtol=1e-5, atol=1e-6)


def test_reference_module_paths_resolve():
    import waternet.data as d
    import waternet.net as n
    import waternet.training_utils as tu
    for name in ("WaterNet", "ConfidenceMapGenerator", "Refiner"):
        assert hasattr(n, name)
    for name in ("transform", "white_balance_transform", "gamma_correction", "histeq"):
        assert hasattr(d, name)
    for name in ("UIEBDataset", "arr2ten", "ten2arr"):
        assert hasattr(tu, name)
    import hubconf
    assert callable(hubconf.waternet) and "torch" in hubconf.dependencies


def test_mode_constants_match_the_header():
    """include/waternet_b200.h and the ctypes binding agree on the forward modes."""
    import re
    from waternet_b200 import _lib
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                             "waternet_b200.h")).read()
    defs = {m.group(1): int(m.group(2).strip("()")) for m in
            re.finditer(r"#define\s+WN_MODE_(\w+)\s+(\(?-?\d+\)?)", text)}
    assert defs == {"FP32_SIMT": _lib.MODE_FP32_SIMT, "BF16X3": _lib.MODE_BF16X3, "BF16_FP8": _lib.MODE_BF16_FP8,
                    "DEFAULT": _lib.MODE_DEFAULT}
