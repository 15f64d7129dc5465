"""The 8 x 24-pixel tiles of the tensor-core convolutions that run three consumer warpgroups (kSpecs wgs = 3), at the
shapes they add: heights around multiples of 24 (1, 23, 24, 25, 47, 49, 71, 1080) against widths around multiples of 8
(1, 7, 8, 9, 17), in both tensor-core modes.  Every launch is checked against float64 on its own input with the bars
of test_forward_layers_gpu.py; the tiled and ragged enhance paths, with windows that are not multiples of 24, must give
the whole-image bits.  When the WN_UMMA_WGS2 library (every layer on 8 x 16 tiles) has been built next to the product
library, the debug dumps of the launches must be bitwise equal between the two: the tile height moves work between
warpgroups, never what an output element adds up."""
import os
import subprocess
import sys

import pytest
import torch

import forward_reference as fr
from test_conv_tiles_gpu import _frames, _model
from test_forward_layers_gpu import _check_case

pytestmark = pytest.mark.gpu

TC_MODES = ["bf16x3", "bf16_fp8"]
HEIGHTS = [1, 23, 24, 25, 47, 49, 71, 1080]
WIDTHS = [1, 7, 8, 9, 17]
# a batch of two at every other shape
SHAPES = [(1 + (i + j) % 2, h, w) for i, h in enumerate(HEIGHTS) for j, w in enumerate(WIDTHS)]
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
WGS2_LIB = os.path.join(ROOT, "waternet_b200", "libwaternet_b200_wgs2.so")


def _model_sd(sd, precision):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("mode", TC_MODES)
def test_every_launch_at_24_row_tile_edges(mode):
    """Stress weights, random floats: every launch and the gated output against float64 at each shape."""
    sd = fr.weight_set("stress", 11)
    m = _model_sd(sd, mode)
    worst = {}
    for n, h, w in SHAPES:
        _check_case(m, sd, mode, fr.make_inputs("floats", n, h, w, h * 1000 + w), worst, f"{(n, h, w)}")


@pytest.mark.parametrize("precision", TC_MODES)
def test_tiled_enhance_bitwise_with_windows_off_24(precision):
    """enhance_tiled with window extents that are not multiples of 24 gives the untiled call's bits."""
    m = _model(precision)
    eng = m.engine()
    mode = m._mode()
    for (h, w), tile in [((121, 203), (37, 53)), ((95, 140), (23, 29)), ((73, 66), (25, 47))]:
        x = torch.stack(_frames([(h, w)] * 2, h))
        f_a = torch.empty(2, 3, h, w, device="cuda")
        f_b = torch.full((2, 3, h, w), float("nan"), device="cuda")
        u_a = eng.enhance(x, mode=mode, out_f32=f_a)
        u_b = eng.enhance_tiled(x, tile=tile, mode=mode, out_f32=f_b, max_pass_pixels=20_000)
        torch.cuda.synchronize()
        assert not eng.f8_overflowed()
        assert torch.equal(u_a, u_b), ((h, w), tile)
        assert torch.equal(f_a, f_b), ((h, w), tile)


@pytest.mark.parametrize("precision", TC_MODES)
def test_ragged_enhance_bitwise_at_24_row_edges(precision):
    """A ragged call over images whose sizes and windows are not multiples of 24 gives each image's bits alone."""
    m = _model(precision)
    eng = m.engine()
    mode = m._mode()
    sizes = [(1, 1), (23, 7), (24, 8), (25, 9), (47, 17), (49, 40), (71, 53), (97, 118)]
    images = _frames(sizes, 70)
    want_u8, want_f32 = [], []
    for img in images:
        f = torch.empty(1, 3, img.shape[0], img.shape[1], device="cuda")
        want_u8.append(eng.enhance(img[None], mode=mode, out_f32=f)[0])
        want_f32.append(f)
    got_f32 = [torch.full_like(f, float("nan")) for f in want_f32]
    got_u8 = eng.enhance_ragged(images, tile=(43, 61), mode=mode, out_f32=got_f32, max_pass_pixels=30_000)
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    for i, (h, w) in enumerate(sizes):
        assert torch.equal(want_u8[i], got_u8[i]), (h, w)
        assert torch.equal(want_f32[i], got_f32[i]), (h, w)


# run in a process of its own per library: the binding loads one library per process (WATERNET_B200_LIB)
_DUMP = r"""
import sys, torch
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import forward_reference as fr
from waternet_b200.net import WaterNet
out = {}
for mode in ("bf16x3", "bf16_fp8"):
    sd = fr.weight_set("stress", 11)
    m = WaterNet(precision=mode)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().eval()
    eng = m.engine()
    for n, h, w in ((2, 37, 53), (1, 300, 500), (1, 1080, 1920)):
        ins = [t.cuda() for t in fr.make_inputs("floats", n, h, w, h * 1000 + w)]
        for layer in range(11):
            out[(mode, n, h, w, layer)] = eng.debug_layer(*ins, layer=layer, mode=m._mode()).cpu()
        with torch.no_grad():
            out[(mode, n, h, w, "out")] = m(*ins).cpu()
torch.save(out, sys.argv[3])
"""


def _dump(lib, path):
    env = dict(os.environ, WATERNET_B200_LIB=lib)
    res = subprocess.run([sys.executable, "-c", _DUMP, ROOT, TESTS, path], env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return torch.load(path)


@pytest.mark.skipif(not os.path.exists(WGS2_LIB), reason="the WN_UMMA_WGS2 library has not been built")
def test_launches_bitwise_equal_to_two_warpgroup_tiles(tmp_path):
    """Every debug-layer dump and the forward output: the product library and the WN_UMMA_WGS2 library agree bitwise."""
    prod = _dump(os.path.join(ROOT, "waternet_b200", "libwaternet_b200.so"), str(tmp_path / "product.pt"))
    ref = _dump(WGS2_LIB, str(tmp_path / "wgs2.pt"))
    assert prod.keys() == ref.keys()
    for k in ref:
        assert torch.equal(prod[k], ref[k]), k
