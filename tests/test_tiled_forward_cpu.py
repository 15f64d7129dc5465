"""Tiled forward of fp32 tensors (wn_forward_tiled, wn_confidence_maps_tiled, wn_refine_tiled) without a GPU: the
workspace bound, the rejected arguments, and the ``tile`` attribute of the model and of ``hub.waternet``."""
import copy
import inspect
import io

import pytest
import torch

BYTES_PER_PIXEL = 1868           # kUmmaBytesPerPixel: one pass of the tensor-core forward
REFINED_BYTES_PER_PIXEL = 36     # the three refined images of one pass (sub-modules)
DEFAULT_PASS = 8 << 20           # max_pass_pixels = 0
SLACK = 64 << 10
MODE_DEFAULT, MODE_FP32, MODE_BF16X3, MODE_BF16_FP8 = -1, 0, 1, 2

SIZES = [(64, 64), (300, 520), (1080, 1920), (2160, 3840), (4320, 7680), (5504, 8256), (20000, 30000)]


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def _both(lib):
    return (("forward", lib.wn_forward_tiled_workspace_bytes, 0),
            ("submodule", lib.wn_submodule_tiled_workspace_bytes, REFINED_BYTES_PER_PIXEL))


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("h,w", SIZES)
def test_tiled_forward_workspace_is_bounded_by_one_pass(lib, n, h, w):
    for name, fn, extra in _both(lib):
        for max_pass in (0, 1 << 20, 3 << 20, 32 << 20):
            got = fn(n, h, w, 998, 998, max_pass, MODE_DEFAULT)
            bound = (max_pass or DEFAULT_PASS) * (BYTES_PER_PIXEL + extra) + SLACK
            assert 0 < got <= bound, (name, n, h, w, max_pass, got, bound)
            assert fn(n, h, w, 998, 998, max_pass, MODE_BF16X3) == got
            assert fn(n, h, w, 998, 998, max_pass, MODE_BF16_FP8) == got


def test_submodule_workspace_holds_the_refined_images(lib):
    for h, w in SIZES:
        fwd = lib.wn_forward_tiled_workspace_bytes(1, h, w, 998, 998, 0, MODE_DEFAULT)
        sub = lib.wn_submodule_tiled_workspace_bytes(1, h, w, 998, 998, 0, MODE_DEFAULT)
        assert fwd < sub <= fwd * (BYTES_PER_PIXEL + REFINED_BYTES_PER_PIXEL) / BYTES_PER_PIXEL + 1024


def test_workspace_does_not_grow_with_the_image(lib):
    a = lib.wn_forward_tiled_workspace_bytes(1, 4320, 7680, 998, 998, 0, MODE_DEFAULT)
    b = lib.wn_forward_tiled_workspace_bytes(1, 20000, 30000, 998, 998, 0, MODE_DEFAULT)
    assert b <= a * 1.1


def test_45_mp_photo_fits_in_16_gb(lib):
    assert lib.wn_forward_tiled_workspace_bytes(1, 5504, 8256, 998, 998, 0, MODE_DEFAULT) <= 16e9
    assert lib.wn_submodule_tiled_workspace_bytes(1, 5504, 8256, 998, 998, 0, MODE_DEFAULT) <= 16e9
    assert lib.wn_forward_workspace_bytes(1, 5504, 8256, MODE_DEFAULT) > 80e9  # what the untiled call would need


def test_bad_arguments_give_no_workspace(lib):
    for name, fn, _ in _both(lib):
        assert fn(1, 64, 64, 32, 32, 0, MODE_DEFAULT) > 0
        for args in [(0, 64, 64, 32, 32, 0, MODE_DEFAULT), (1, 0, 64, 32, 32, 0, MODE_DEFAULT),
                     (1, 64, -1, 32, 32, 0, MODE_DEFAULT), (1, 64, 64, 0, 32, 0, MODE_DEFAULT),
                     (1, 64, 64, 32, -5, 0, MODE_DEFAULT), (1, 64, 64, 32, 32, -1, MODE_DEFAULT),
                     (1, 64, 64, 32, 32, 0, MODE_FP32), (1, 64, 64, 32, 32, 0, 7),
                     (65536, 64, 64, 32, 32, 0, MODE_DEFAULT),
                     (1, 30000, 30000, 998, 998, 0, MODE_DEFAULT)]:  # over the size limit (~715 Mpx)
            assert fn(*args) == 0, (name, args)


def test_null_arguments_fail_with_a_message(lib):
    assert lib.wn_forward_tiled(None, None, None, None, None, None, None, 1, 64, 64, 32, 32, 0, MODE_DEFAULT, None, 0,
                                None) != 0
    assert b"wn_forward_tiled: null" in lib.wn_last_error()
    assert lib.wn_confidence_maps_tiled(None, None, None, None, None, None, None, 1, 64, 64, 32, 32, 0, MODE_DEFAULT,
                                        None, 0, None) != 0
    assert b"wn_confidence_maps_tiled: null" in lib.wn_last_error()
    assert lib.wn_refine_tiled(None, 0, None, None, None, None, 1, 64, 64, 32, 32, 0, MODE_DEFAULT, None, 0,
                               None) != 0
    assert b"wn_refine_tiled: null" in lib.wn_last_error()


def test_tile_attribute_survives_deepcopy_and_pickling():
    from oracle import forward as ofw
    from waternet_b200.net import WaterNet
    plain = WaterNet()
    m = WaterNet(tile=(64, 96))
    m.load_state_dict(ofw.synthetic_state_dict(0))
    assert plain.tile is None and m.tile == (64, 96)
    assert list(m.state_dict().keys()) == list(plain.state_dict().keys())
    twin = copy.deepcopy(m)
    assert twin.tile == (64, 96) and twin.cmg._parent_ref() is twin
    buf = io.BytesIO()
    torch.save(m, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert again.tile == (64, 96) and again.gc_refiner._parent_ref() is again
    for k, v in m.state_dict().items():
        assert torch.equal(again.state_dict()[k], v)
    m.tile = 998
    assert copy.deepcopy(m).tile == 998


def test_tile_is_a_plain_attribute_of_free_standing_stacks():
    from waternet_b200.net import ConfidenceMapGenerator, Refiner
    cmg, ref = ConfidenceMapGenerator(), Refiner()
    assert cmg.tile is None and ref.tile is None
    cmg.tile = 128
    assert copy.deepcopy(cmg).tile == 128 and Refiner().tile is None


def test_tile_with_the_fp32_precision_is_refused():
    from waternet_b200.net import WaterNet
    with pytest.raises(ValueError, match="tensor cores"):
        WaterNet(precision="fp32", tile=64)
    with pytest.raises(ValueError):
        WaterNet(tile=0)
    m = WaterNet(precision="fp32")
    m.tile = 64
    with torch.no_grad(), pytest.raises(ValueError, match="tensor cores"):
        m(*[torch.rand(1, 3, 8, 8) for _ in range(4)])


def test_hub_waternet_accepts_tile():
    from waternet_b200 import hub
    params = inspect.signature(hub.waternet).parameters
    assert list(params)[:2] == ["pretrained", "device"]  # the reference's positional use is unchanged
    assert "tile" in params and params["tile"].default is None
    if torch.cuda.is_available():
        pytest.skip("CUDA present: the GPU tests run the model")
    from waternet_b200 import WaterNetLibraryError
    with pytest.raises(WaterNetLibraryError, match="CUDA"):  # no TypeError: the keyword is accepted
        hub.waternet(pretrained=False, tile=998)
