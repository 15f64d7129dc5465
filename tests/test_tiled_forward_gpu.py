"""Tiled forward of fp32 tensors (wn_forward_tiled, wn_confidence_maps_tiled, wn_refine_tiled) on the GPU:
bit-identical to the untiled calls, and right where the untiled call cannot run (a 45 MP photo needs 85 GB
untiled)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import forward as ofw
from oracle import preprocess as opre

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
MODE = {"bf16x3": 1, "bf16_fp8": 2, "default": -1}


def _model(sd, precision="default", tile=None):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision, tile=tile)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _frames(n, h, w, seed=0):
    return torch.from_numpy(np.stack([ofw.synthetic_image(seed + i, h, w, "smooth" if i % 2 else "noise")
                                      for i in range(n)])).cuda()


def _levels(n, h, w, seed=0):
    """The four inputs as the reference's preprocess makes them: 8-bit levels / 255."""
    from waternet_b200.engine import get_engine
    pre = get_engine().preprocess(_frames(n, h, w, seed))
    return [pre[k] for k in ("x", "wb", "he", "gc")]


def _rand(n, h, w, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand((n, 3, h, w), generator=g, device="cuda") for _ in range(4)]


def _nan_like(t):
    return torch.full(t.shape, float("nan"), device=t.device)


def _assert_bitwise(a, b, what):
    assert torch.equal(a, b), f"{what}: {int((a != b).sum())} of {a.numel()} values differ"
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), what


def _forward_tiled_ff(eng, ins, tile, mode, max_pass_pixels=0):
    """wn_forward_tiled into a NaN-filled output with a workspace of 0xFF bytes."""
    n, _, h, w = ins[0].shape
    th, tw = eng._tile_hw(tile)
    nbytes = eng.forward_tiled_workspace_bytes(n, h, w, tile, mode, max_pass_pixels)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    out = torch.full((n, 3, h, w), float("nan"), device="cuda")
    strides = (ctypes.c_int64 * 16)(*[s for t in ins for s in t.stride()])
    rc = eng.lib.wn_forward_tiled(eng.handle, *[t.data_ptr() for t in ins], strides, out.data_ptr(), n, h, w, th, tw,
                                  max_pass_pixels, mode, ws.data_ptr(), ws.numel(),
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    from waternet_b200 import _lib
    _lib.check(rc, "wn_forward_tiled")
    return out


def _assert_same(eng, ins, mode, tile, max_pass_pixels=0):
    """forward_tiled == forward, bitwise; the e4m3 range flag stays down."""
    want = eng.forward(*ins, mode=mode)
    got = eng.forward_tiled(*ins, tile=tile, mode=mode, out=_nan_like(want), max_pass_pixels=max_pass_pixels)
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    _assert_bitwise(got, want, "forward_tiled")
    return want


@pytest.mark.parametrize("inputs", ["levels", "rand"])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16_fp8"])
def test_forward_tiled_equals_forward_over_several_passes(precision, inputs):
    """3 x 300x520, tile 64x96: 90 windows of 113x86, 40 per pass -> passes of 40, 40 and 10.  Levels take the
    2-pass first layer, torch.rand inputs the general 3-pass one."""
    from waternet_b200.engine import tile_geometry
    m = _model(ofw.synthetic_state_dict(0, 3.0), precision)
    eng = m.engine()
    g = tile_geometry(300, 520, 64, 96)
    max_pass = 40 * g["win_h"] * g["win_w"] + 5
    ins = _levels(3, 300, 520) if inputs == "levels" else _rand(3, 300, 520)
    want = _assert_same(eng, ins, MODE[precision], (64, 96), max_pass)
    _assert_bitwise(_forward_tiled_ff(eng, ins, (64, 96), MODE[precision], max_pass), want, "0xFF workspace")


@pytest.mark.parametrize("h,w,tile", [
    (37, 53, (256, 256)),    # the image is smaller than one window
    (40, 700, (128, 128)),   # one axis smaller than the window
    (113, 117, (32, 32)),    # sizes that are not multiples of 8
    (192, 256, (64, 128)),   # the tile divides the image exactly
    (50, 70, (8, 8)),        # tile 8: windows of 34 x 34
])
def test_forward_tiled_equals_forward_edge_shapes(h, w, tile):
    m = _model(ofw.synthetic_state_dict(3, 3.0))
    _assert_same(m.engine(), _levels(2, h, w, seed=10), MODE["default"], tile)
    _assert_same(m.engine(), _rand(2, h, w, seed=11), MODE["default"], tile)


def test_forward_tiled_reads_channels_last_and_sliced_inputs():
    """Each input with strides of its own: channels_last (what arr2ten produces), a crop of a larger tensor, a
    channel slice of a wider one and every other image of a larger batch."""
    n, h, w = 2, 150, 230
    m = _model(ofw.synthetic_state_dict(1, 3.0))
    eng = m.engine()
    base = _levels(n, h, w, seed=20)
    x = base[0].contiguous(memory_format=torch.channels_last)
    big = torch.rand(n, 3, h + 9, w + 17, device="cuda")
    big[:, :, 4:4 + h, 7:7 + w] = base[1]
    wb = big[:, :, 4:4 + h, 7:7 + w]
    wide = torch.rand(n, 8, h, w, device="cuda")
    wide[:, 2:5] = base[2]
    he = wide[:, 2:5]
    batch = torch.rand(2 * n, 3, h, w, device="cuda")
    batch[::2] = base[3]
    gc = batch[::2]
    ins = [x, wb, he, gc]
    assert len({t.stride() for t in ins}) == 4 and not any(t.is_contiguous() for t in ins)
    for mode in (MODE["bf16x3"], MODE["default"]):
        want = eng.forward(*base, mode=mode)
        got = eng.forward_tiled(*ins, tile=(48, 64), mode=mode, out=_nan_like(want), max_pass_pixels=20000)
        _assert_bitwise(got, want, f"strided inputs, mode {mode}")


def _nudged_batch(h, w):
    """Two images of 8-bit levels; in the second one value is moved off its level."""
    ins = [t.clone() for t in _levels(2, h, w, seed=30)]
    ins[2][1, 1, h // 2, w // 3] += 1e-3
    return ins


@pytest.mark.parametrize("precision", ["bf16x3", "bf16_fp8"])
def test_exact_levels_flag_is_taken_over_the_whole_call(precision):
    """One image of levels and one with a value nudged off a level: the flag is down for the call, as for the
    untiled call that runs the batch in one pass.  With one image per untiled pass the levels image takes the 2-pass
    first layer untiled and the 3-pass one tiled; the a_lo pass adds exact zeros, so the bits agree."""
    h, w = 200, 260
    m = _model(ofw.synthetic_state_dict(2, 3.0), precision)
    eng = m.engine()
    ins = _nudged_batch(h, w)
    assert eng.chunk_images(2, h, w) == 2
    _assert_same(eng, ins, MODE[precision], (64, 64), max_pass_pixels=30000)
    try:
        eng.set_chunk_pixels(h * w)
        assert eng.chunk_images(2, h, w) == 1
        _assert_same(eng, ins, MODE[precision], (64, 64), max_pass_pixels=30000)
    finally:
        eng.set_chunk_pixels(0)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16_fp8"])
def test_submodules_tiled_equal_untiled(precision):
    """The engine calls over several passes, the children of a WaterNet(tile=...) and free-standing modules."""
    from waternet_b200.net import ConfidenceMapGenerator, Refiner
    sd = ofw.synthetic_state_dict(4, 3.0)
    mode = MODE[precision]
    plain, tiled = _model(sd, precision), _model(sd, precision, tile=(64, 96))
    eng = plain.engine()
    for ins in (_levels(2, 300, 520, seed=40), _rand(2, 300, 520, seed=41)):
        want = eng.confidence_maps(*ins, mode=mode)
        _assert_bitwise(eng.confidence_maps_tiled(*ins, tile=(64, 96), mode=mode, max_pass_pixels=50000), want,
                        "confidence_maps_tiled")
        for which in range(3):
            want = eng.refine(which, ins[0], ins[1 + which], mode=mode)
            got = eng.refine_tiled(which, ins[0], ins[1 + which], tile=(64, 96), mode=mode, max_pass_pixels=50000)
            _assert_bitwise(got, want, f"refine_tiled({which})")
        with torch.no_grad():
            _assert_bitwise(torch.cat(tiled.cmg(*ins), 1), torch.cat(plain.cmg(*ins), 1), "WaterNet(tile).cmg")
            for name, xbar in zip(("wb_refiner", "ce_refiner", "gc_refiner"), ins[1:]):
                _assert_bitwise(getattr(tiled, name)(ins[0], xbar), getattr(plain, name)(ins[0], xbar),
                                f"WaterNet(tile).{name}")
            _assert_bitwise(tiled(*ins), plain(*ins), "WaterNet(tile)")
    free_cmg, free_ref = ConfidenceMapGenerator().cuda().eval(), Refiner().cuda().eval()
    free_cmg.load_state_dict({k[4:]: v for k, v in sd.items() if k.startswith("cmg.")})
    free_ref.load_state_dict({k[11:]: v for k, v in sd.items() if k.startswith("ce_refiner.")})
    free_cmg.precision = free_ref.precision = precision
    ins = _levels(1, 180, 300, seed=42)
    with torch.no_grad():
        want_maps, want_ref = torch.cat(free_cmg(*ins), 1), free_ref(ins[0], ins[2])
        free_cmg.tile = free_ref.tile = 48
        _assert_bitwise(torch.cat(free_cmg(*ins), 1), want_maps, "free-standing cmg")
        _assert_bitwise(free_ref(ins[0], ins[2]), want_ref, "free-standing refiner")


def test_45_mp_photo_through_the_hub_model_against_the_oracle_on_crops():
    """hub.waternet(tile=998): preprocess -> model -> postprocess on one 8256x5504 photo (untiled: 85 GB of
    workspace).  The output on crops at the corners, the borders, tile seams and the interior against the CPU oracle,
    each crop run with 13 pixels of context; and bit for bit what enhance_tiled computes from the same photo."""
    from waternet_b200 import hub
    from waternet_b200.engine import TILE_HALO, tile_geometry
    h, w = 5504, 8256
    sd = ofw.synthetic_state_dict(0, 3.0)
    preprocess, postprocess, model = hub.waternet(pretrained=False, tile=998)
    model.load_state_dict(sd)
    model.eval()
    assert model.tile == 998
    eng = model.engine()
    assert eng.forward_tiled_workspace_bytes(1, h, w, 998) < 16e9
    rgb = ofw.synthetic_image(60, h, w, "noise")
    try:
        ins = preprocess(rgb)
        with torch.no_grad():
            out = model(*ins)
        u8 = postprocess(out)
        torch.cuda.synchronize()
        assert not eng.f8_overflowed()
        eng.release_workspaces()
        f32 = torch.full((1, 3, h, w), float("nan"), device="cuda")
        u8_e = eng.enhance_tiled(torch.from_numpy(rgb[None]).cuda(), tile=998, out_f32=f32)
        _assert_bitwise(out, f32, "model(tile=998) against enhance_tiled")
        assert np.array_equal(u8, u8_e.cpu().numpy())
        ins = [t.cpu() for t in ins]
        out = out.cpu().numpy()
    finally:
        eng.release_workspaces()
    g = tile_geometry(h, w, 998, 998)
    sy, sx = 2 * g["th"], 4 * g["tw"]  # a seam row / column
    s = 24
    crops = [(0, 0), (0, w - s), (h - s, 0), (h - s, w - s),      # corners
             (0, sx - s // 2), (sy - s // 2, 0),                    # borders across a seam
             (h - s, sx - s // 2), (sy - s // 2, w - s),
             (sy - s // 2, sx - s // 2),                            # a seam crossing
             (g["th"] + 300, g["tw"] + 300)]                        # the interior of a tile
    for y0, x0 in crops:
        a0, a1 = max(0, y0 - TILE_HALO), min(h, y0 + s + TILE_HALO)
        b0, b1 = max(0, x0 - TILE_HALO), min(w, x0 + s + TILE_HALO)
        ref = ofw.waternet_forward(sd, *[t[:, :, a0:a1, b0:b1] for t in ins]).numpy()
        ref = ref[:, :, y0 - a0:y0 - a0 + s, x0 - b0:x0 - b0 + s]
        got = out[:, :, y0:y0 + s, x0:x0 + s]
        err = np.max(np.abs(got - ref))
        assert err <= REL_TOL * np.max(np.abs(ref)), (y0, x0, err)
        du8 = np.abs(u8[0, y0:y0 + s, x0:x0 + s].astype(int) - opre.ten2arr(ref)[0].astype(int))
        assert du8.max() <= 1, (y0, x0)


def test_range_guard_rerun_on_the_tiled_forward():
    """Weights whose activations leave the e4m3 range: the default mode recomputes every pass with the bf16x3
    kernels, so its output equals the bf16x3 output bit for bit."""
    sd = ofw.synthetic_state_dict(0, 3.0)
    sd["wb_refiner.conv1.weight"] = sd["wb_refiner.conv1.weight"] * 400.0
    sd["wb_refiner.conv2.weight"] = sd["wb_refiner.conv2.weight"] / 400.0
    ins = _levels(2, 120, 200, seed=30)
    f8, plain = _model(sd, "default"), _model(sd, "bf16x3")
    a = f8.engine().forward_tiled(*ins, tile=48, mode=MODE["default"], out=_nan_like(ins[0]), max_pass_pixels=10000)
    b = plain.engine().forward_tiled(*ins, tile=48, mode=MODE["bf16x3"], out=_nan_like(ins[0]),
                                     max_pass_pixels=10000)
    torch.cuda.synchronize()
    assert f8.engine().f8_overflowed()
    _assert_bitwise(a, b, "range guard")


def test_forward_tiled_in_a_cuda_graph():
    m = _model(ofw.synthetic_state_dict(5, 3.0))
    eng = m.engine()
    ins = _rand(2, 130, 170, seed=50)
    want = eng.forward_tiled(*ins, tile=(40, 56), max_pass_pixels=12000)  # warm-up: workspace, encoder, attributes
    out = torch.empty_like(want)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eng.forward_tiled(*ins, tile=(40, 56), out=out, max_pass_pixels=12000)
    out.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    _assert_bitwise(out, want, "graph replay")


def test_tile_is_ignored_when_autograd_records():
    sd = ofw.synthetic_state_dict(6, 3.0)
    plain, tiled = _model(sd), _model(sd, tile=16)
    outs, grads = [], []
    for m in (plain, tiled):
        ins = [t.clone().requires_grad_(True) for t in _levels(2, 40, 48, seed=60)]
        out = m(*ins)
        out.backward(torch.linspace(-1, 1, out.numel(), device="cuda").view_as(out))
        outs.append(out.detach())
        grads.append([p.grad for p in m.parameters()] + [t.grad for t in ins])
    _assert_bitwise(outs[1], outs[0], "output with a graph")
    for a, b in zip(grads[1], grads[0]):
        _assert_bitwise(a, b, "gradient")
