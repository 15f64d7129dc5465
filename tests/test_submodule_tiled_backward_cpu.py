"""Windowed recompute backward of one sub-module (wn_confidence_maps_backward_tiled, wn_refine_backward_tiled) without
a GPU: the workspace bound, the rejected arguments, null pointers, and the ``grad_tile`` attribute of the stacks."""
import copy
import ctypes
import io

import pytest
import torch

from oracle import forward as ofw

CMG_BYTES_PER_PIXEL = 3852                      # carve(kStackCmg): the cmg's activations and gradient buffers
REFINER_BYTES_PER_PIXEL = 1828                  # carve(kStackRefiners)
DEFAULT_PASS = 2 << 20                          # max_pass_pixels = 0
MAX_PASS = 8 << 20                              # kTrainMaxPixels
DENSE_BYTES = 49 * 128 * 128 * 4                # kDenseBytes: one layer's weight gradient, dense
PARTIAL_BYTES = 192 * 512 * 128 * 4             # kPartialBytes: per-CTA partial sums of the weight-gradient GEMMs
CMG_SPEC = [(12, 128, 7), (128, 128, 5), (128, 128, 3), (128, 64, 1), (64, 64, 7), (64, 64, 5), (64, 64, 3),
            (64, 3, 3)]
REFINER_SPEC = [(6, 32, 7), (32, 32, 5), (32, 3, 3)]
SIZES = [(64, 64), (300, 520), (1080, 1920), (2160, 3840), (4320, 7680), (5504, 8256), (20000, 30000)]


def _scratch(spec):
    """The scratch copy of a stack's parameter gradients, each tensor rounded up to 256 bytes."""
    return sum(-(-4 * n // 256) * 256 for ci, co, k in spec for n in (co * ci * k * k, co))


STACKS = {0: (CMG_BYTES_PER_PIXEL, _scratch(CMG_SPEC)), 1: (REFINER_BYTES_PER_PIXEL, _scratch(REFINER_SPEC))}


def _fixed(stack):
    return DENSE_BYTES + PARTIAL_BYTES + STACKS[stack][1] + (24 << 10)  # + the flag and every region's alignment


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.mark.parametrize("stack", [0, 1])
@pytest.mark.parametrize("n", [1, 16])
@pytest.mark.parametrize("h,w", SIZES)
def test_workspace_is_bounded_by_one_pass(lib, stack, n, h, w):
    for max_pass in (0, 1 << 20, 4 << 20, MAX_PASS):
        got = lib.wn_submodule_backward_tiled_workspace_bytes(n, h, w, 998, 998, max_pass, stack)
        bound = (max_pass or DEFAULT_PASS) * STACKS[stack][0] + _fixed(stack)
        assert 0 < got <= bound, (stack, n, h, w, max_pass, got, bound)


@pytest.mark.parametrize("stack", [0, 1])
def test_workspace_does_not_grow_with_the_image(lib, stack):
    fn = lib.wn_submodule_backward_tiled_workspace_bytes
    sizes = [fn(1, h, w, 998, 998, 0, stack) for h, w in SIZES[2:]]
    assert max(sizes) <= DEFAULT_PASS * STACKS[stack][0] + _fixed(stack)
    assert fn(16, 1080, 1920, 998, 998, 0, stack) <= max(sizes) * 1.1
    # what the untiled training call would keep for a 45 MP photo: refused, and far more
    assert lib.wn_submodule_train_workspace_bytes(1, 5504, 8256, stack) == 0
    assert 5504 * 8256 * STACKS[stack][0] > 10 * max(sizes)


def test_default_pass_sizes(lib):
    """At the default pass: at most about 8.1 GB for the cmg and 3.9 GB for a refiner, and a refiner needs less than
    half of what the cmg needs once the pass holds more than a few thousand pixels."""
    fn = lib.wn_submodule_backward_tiled_workspace_bytes
    cmg = [fn(1, h, w, 998, 998, 0, 0) for h, w in SIZES[2:]]
    ref = [fn(1, h, w, 998, 998, 0, 1) for h, w in SIZES[2:]]
    assert max(cmg) < 8.2e9 and max(ref) < 3.95e9
    assert all(r < 0.5 * c for r, c in zip(ref, cmg))
    # the sub-module calls need less than the whole network's windowed backward
    whole = lib.wn_backward_tiled_workspace_bytes(1, 5504, 8256, 998, 998, 0)
    assert fn(1, 5504, 8256, 998, 998, 0, 0) < whole and fn(1, 5504, 8256, 998, 998, 0, 1) < 0.4 * whole


def test_bad_arguments_give_no_workspace(lib):
    fn = lib.wn_submodule_backward_tiled_workspace_bytes
    for stack in (0, 1):
        assert fn(1, 64, 64, 32, 32, 0, stack) > 0
        assert fn(1, 64, 64, 32, 32, MAX_PASS, stack) > 0
        assert fn(65535, 8, 8, 8, 8, 0, stack) > 0
        assert fn(1, 2048, 4096, 4096, 4096, 0, stack) > 0  # one 8 Mi-pixel window
        for args in [(0, 64, 64, 32, 32, 0), (-1, 64, 64, 32, 32, 0), (1, 0, 64, 32, 32, 0), (1, 64, -1, 32, 32, 0),
                     (1, 64, 64, 0, 32, 0), (1, 64, 64, 32, -5, 0), (1, 64, 64, 32, 32, -1),
                     (1, 64, 64, 32, 32, MAX_PASS + 1), (65536, 64, 64, 32, 32, 0),
                     (1, 30000, 30000, 998, 998, 0),  # over the size limit (~715 Mpx)
                     (1, 2049, 4096, 4096, 4096, 0),  # a window of more than 8 Mi pixels
                     (1, 3000, 4000, 3000, 4000, 0)]:
            assert fn(*args, stack) == 0, (args, stack)
    for stack in (-1, 2, 3):
        assert fn(1, 64, 64, 32, 32, 0, stack) == 0, stack


def test_null_arguments_fail_with_a_message(lib):
    from waternet_b200 import _lib
    grads = (ctypes.c_void_p * _lib.NUM_PARAMS)()
    assert lib.wn_confidence_maps_backward_tiled(None, None, None, None, None, None, None, grads, None, 1, 64, 64, 32,
                                                 32, 0, None, 0, None) == -1
    assert b"wn_confidence_maps_backward_tiled: null" in lib.wn_last_error()
    assert lib.wn_refine_backward_tiled(None, 0, None, None, None, None, grads, None, 1, 64, 64, 32, 32, 0, None, 0,
                                        None) == -1
    assert b"wn_refine_backward_tiled: null" in lib.wn_last_error()
    for which in (-1, 3):
        assert lib.wn_refine_backward_tiled(None, which, None, None, None, None, grads, None, 1, 64, 64, 32, 32, 0,
                                            None, 0, None) == -1
        assert b"which must be 0, 1 or 2" in lib.wn_last_error()


def test_grad_tile_defaults_to_none_and_survives_deepcopy_and_pickling():
    from waternet_b200.net import ConfidenceMapGenerator, Refiner, WaterNet
    sd = ofw.synthetic_state_dict(0)
    for cls, prefix in ((ConfidenceMapGenerator, "cmg"), (Refiner, "ce_refiner")):
        plain = cls()
        m = cls()
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in sd.items() if k.startswith(prefix + ".")})
        assert plain.grad_tile is None and m.grad_tile is None and m._grad_tile() is None
        m.grad_tile = (64, 96)
        assert m._grad_tile() == (64, 96)
        assert list(m.state_dict().keys()) == list(plain.state_dict().keys())
        assert copy.deepcopy(m).grad_tile == (64, 96)
        buf = io.BytesIO()
        torch.save(m, buf)
        buf.seek(0)
        again = torch.load(buf, weights_only=False)
        assert again.grad_tile == (64, 96)
        del again.__dict__["grad_tile"]  # a stack pickled before the attribute existed
        assert again.grad_tile is None
    net = WaterNet()
    assert all(s._grad_tile() is None for s in (net.cmg, net.wb_refiner, net.ce_refiner, net.gc_refiner))
    net.grad_tile = 40
    assert all(s._grad_tile() == (40, 40) for s in (net.cmg, net.wb_refiner, net.ce_refiner, net.gc_refiner))
    assert net.cmg.grad_tile is None  # a bound stack follows its parent; its own attribute is not touched
    twin = copy.deepcopy(net)
    assert twin.gc_refiner._grad_tile() == (40, 40)


def test_grad_tile_with_the_fp32_precision_is_refused():
    from waternet_b200.net import ConfidenceMapGenerator, Refiner, WaterNet
    ins = [torch.rand(1, 3, 8, 8, requires_grad=True) for _ in range(4)]
    for m, call in ((ConfidenceMapGenerator(), lambda m: m(*ins)), (Refiner(), lambda m: m(ins[0], ins[1]))):
        m.precision = "fp32"
        m.grad_tile = 16
        with pytest.raises(ValueError, match="tensor cores"):
            call(m)
        m.grad_tile = 0
        m.precision = "default"
        with pytest.raises(ValueError):
            call(m)
    net = WaterNet(precision="fp32")
    net.grad_tile = 16
    with pytest.raises(ValueError, match="tensor cores"):
        net.cmg(*ins)
    with pytest.raises(ValueError, match="tensor cores"):
        net.wb_refiner(ins[0], ins[1])


def test_cpu_tensors_keep_the_torch_graph_with_grad_tile():
    from waternet_b200.net import Refiner, WaterNet
    sd = ofw.synthetic_state_dict(3, 3.0)
    net = WaterNet(grad_tile=16)
    net.load_state_dict(sd)
    x, wb, he, gc = [torch.rand(2, 3, 9, 11, generator=torch.Generator().manual_seed(i)) for i in range(4)]
    maps = torch.cat(net.cmg(x, wb, he, gc), 1)
    assert torch.allclose(maps, ofw.confidence_maps(sd, x, wb, he, gc), rtol=1e-5, atol=1e-6)
    maps.sum().backward()
    assert net.cmg.conv1.weight.grad is not None and net.wb_refiner.conv1.weight.grad is None
    free = Refiner()
    free.grad_tile = 16
    free.load_state_dict({k[len("gc_refiner."):]: v for k, v in sd.items() if k.startswith("gc_refiner.")})
    out = free(x, gc)
    assert type(out.grad_fn).__name__ == "ReluBackward0"
