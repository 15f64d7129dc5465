"""The sub-modules under autograd without a GPU: the workspace of wn_submodule_train_workspace_bytes, the arguments the
four calls refuse, and which calls keep the torch graph (CPU tensors, precision "fp32", an image over the limit)."""
import ctypes
import types

import pytest
import torch

from oracle import forward as ofw

DENSE_BYTES = 49 * 128 * 128 * 4        # kDenseBytes: one layer's weight gradient, dense
PARTIAL_BYTES = 192 * 512 * 128 * 4     # kPartialBytes: per-CTA partial sums of the weight-gradient GEMMs
FIXED = DENSE_BYTES + PARTIAL_BYTES + 1024 + 1023  # + the exact-levels flag's 1 KiB region + alignment of the base
# act0 64 | cmg activations 3 x 512 + 4 x 256 | maps 12 | gradient ping-pong 2 x 512 | conv8 seed 64 | input grads 128
CMG_BYTES_PER_PIXEL = 64 + 3 * 512 + 4 * 256 + 12 + 2 * 512 + 64 + 128
# act0 64 | refiner activations 2 x 384 | refined images 36 | gradient ping-pong 2 x 384 | conv3 seed 64 | input grads
REFINER_BYTES_PER_PIXEL = 64 + 2 * 384 + 36 + 2 * 384 + 64 + 128
MAX_PIXELS = 8 << 20


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.mark.parametrize("n,h,w", [(1, 16, 16), (16, 112, 112), (2, 1080, 1920), (1, 2048, 4096), (32768, 16, 16)])
def test_workspace_is_the_stack_alone(lib, n, h, w):
    """Pixel counts that are multiples of 256 leave no region padding: the size is exact."""
    px = n * h * w
    assert lib.wn_submodule_train_workspace_bytes(n, h, w, 0) == px * CMG_BYTES_PER_PIXEL + FIXED
    assert lib.wn_submodule_train_workspace_bytes(n, h, w, 1) == px * REFINER_BYTES_PER_PIXEL + FIXED
    if px >= 1 << 20:  # a refiner keeps about a third of what the whole network keeps, the cmg about 70 %
        assert lib.wn_submodule_train_workspace_bytes(n, h, w, 1) < 0.35 * lib.wn_train_workspace_bytes(n, h, w)
        assert lib.wn_submodule_train_workspace_bytes(n, h, w, 0) < 0.7 * lib.wn_train_workspace_bytes(n, h, w)


def test_the_image_limit_is_accepted(lib):
    for stack in (0, 1):
        assert lib.wn_submodule_train_workspace_bytes(65535, 1, 1, stack) > 0
        assert lib.wn_submodule_train_workspace_bytes(1, 2048, 4096, stack) > 0


def test_odd_sizes_round_every_region_up(lib):
    for stack, per_px in ((0, CMG_BYTES_PER_PIXEL), (1, REFINER_BYTES_PER_PIXEL)):
        got = lib.wn_submodule_train_workspace_bytes(3, 1, 1, stack)
        assert 3 * per_px + FIXED <= got <= 3 * per_px + FIXED + 16 * 1024


def test_rejected_arguments_give_no_workspace(lib):
    fn = lib.wn_submodule_train_workspace_bytes
    for args in [(1, 8, 8, 2), (1, 8, 8, -1), (0, 8, 8, 0), (-1, 8, 8, 1), (1, 0, 8, 0), (1, 8, -3, 1),
                 (65536, 1, 1, 0), (65536, 1, 1, 1),          # more than 65535 images
                 (1, 2048, 4097, 0), (3, 2048, 2048, 1),      # more than 8 Mi pixels
                 (1 << 30, 1 << 16, 1 << 16, 1)]:
        assert fn(*args) == 0, args


def test_null_and_out_of_range_arguments_fail_with_a_message(lib):
    from waternet_b200 import _lib
    grads = (ctypes.c_void_p * _lib.NUM_PARAMS)()
    assert lib.wn_confidence_maps_train(None, None, None, None, None, None, None, 1, 8, 8, None, 0, None) == -1
    assert b"wn_confidence_maps_train: null" in lib.wn_last_error()
    assert lib.wn_confidence_maps_backward(None, None, grads, None, 1, 8, 8, None, 0, None) == -1
    assert b"wn_confidence_maps_backward: null" in lib.wn_last_error()
    assert lib.wn_refine_train(None, 0, None, None, None, None, 1, 8, 8, None, 0, None) == -1
    assert b"wn_refine_train: null" in lib.wn_last_error()
    assert lib.wn_refine_backward(None, 0, None, grads, None, 1, 8, 8, None, 0, None) == -1
    assert b"wn_refine_backward: null" in lib.wn_last_error()
    for which in (-1, 3):
        assert lib.wn_refine_train(None, which, None, None, None, None, 1, 8, 8, None, 0, None) == -1
        assert b"which must be 0, 1 or 2" in lib.wn_last_error()
        assert lib.wn_refine_backward(None, which, None, grads, None, 1, 8, 8, None, 0, None) == -1
        assert b"which must be 0, 1 or 2" in lib.wn_last_error()


def _model(precision="default"):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(ofw.synthetic_state_dict(3, 3.0))
    return m


def test_cpu_tensors_keep_the_torch_graph():
    from waternet_b200.net import Refiner
    m = _model()
    sd = m.state_dict()
    x, wb, he, gc = [torch.rand(2, 3, 9, 11, generator=torch.Generator().manual_seed(i)) for i in range(4)]
    maps = m.cmg(x, wb, he, gc)
    assert torch.allclose(torch.cat(maps, 1), ofw.confidence_maps(sd, x, wb, he, gc), rtol=1e-5, atol=1e-6)
    torch.cat(maps, 1).sum().backward()
    assert m.cmg.conv1.weight.grad is not None and m.wb_refiner.conv1.weight.grad is None
    free = Refiner()
    free.load_state_dict({k[len("gc_refiner."):]: v for k, v in sd.items() if k.startswith("gc_refiner.")})
    out = free(x, gc)
    assert type(out.grad_fn).__name__ == "ReluBackward0"
    assert torch.allclose(out, ofw.refine(sd, "gc_refiner", x, gc), rtol=1e-5, atol=1e-6)


def test_fp32_precision_and_oversize_images_choose_the_torch_graph():
    """The dispatch rule of _train_engine, which a call with autograd recording consults before any device work:
    None (the torch graph) for precision "fp32" and for one image over Engine.TRAIN_MAX_PIXELS."""
    from waternet_b200.engine import Engine
    from waternet_b200.net import ConfidenceMapGenerator, Refiner
    on_cuda = types.SimpleNamespace(is_cuda=True, shape=(1, 3, 64, 64))
    assert _model("fp32").cmg._train_engine(on_cuda) is None
    assert _model("fp32").ce_refiner._train_engine(on_cuda) is None
    for free in (ConfidenceMapGenerator(), Refiner()):
        free.precision = "fp32"
        assert free._train_engine(on_cuda) is None
    huge = types.SimpleNamespace(is_cuda=True, shape=(1, 3, 4096, 2049))
    assert 4096 * 2049 > Engine.TRAIN_MAX_PIXELS
    assert _model().gc_refiner._train_engine(huge) is None
    assert Refiner()._train_engine(huge) is None
    cpu = types.SimpleNamespace(is_cuda=False, shape=(1, 3, 8, 8))
    assert _model().cmg._train_engine(cpu) is None
