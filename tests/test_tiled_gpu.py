"""Tiled enhance (wn_enhance_u8_tiled) on the GPU: bit-identical to the untiled call, and right where the untiled
call cannot run (an 8K frame needs 62 GB untiled)."""
import numpy as np
import pytest
import torch

from oracle import forward as ofw
from oracle import preprocess as opre

pytestmark = pytest.mark.gpu

REL_TOL = 1e-3
MODE = {"bf16x3": 1, "bf16_fp8": 2, "default": -1}


def _model(sd, precision="default"):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _frames(n, h, w, seed=0):
    return torch.from_numpy(np.stack([ofw.synthetic_image(seed + i, h, w, "smooth" if i % 2 else "noise")
                                      for i in range(n)])).cuda()


def _where(diff, h, w, tile):
    """Where a (N, H, W) mismatch mask lies: at window seams (a geometry bug) or spread across the image."""
    from waternet_b200.engine import tile_geometry
    g = tile_geometry(h, w, *tile)
    seams_y = np.array([k0 for _, _, (k0, _), _ in g["windows"] if k0 > 0] or [-99])
    seams_x = np.array([k0 for _, _, _, (k0, _) in g["windows"] if k0 > 0] or [-99])
    idx = np.argwhere(diff)
    dy = np.abs(idx[:, 1, None] - seams_y[None]).min(1)
    dx = np.abs(idx[:, 2, None] - seams_x[None]).min(1)
    near = int(((dy <= 2) | (dx <= 2)).sum())
    return (f"{len(idx)} pixels differ, {near} of them within 2 px of a window seam "
            f"({'seams: a geometry bug' if near * 2 > len(idx) else 'spread across the image'}); "
            f"first (image, y, x): {tuple(idx[0])}")


def _assert_same(eng, frames, mode, tile, max_pass_pixels=0):
    """enhance_tiled == enhance, bitwise, on out_u8 and out_f32; the e4m3 range flag stays down in both runs."""
    n, h, w, _ = frames.shape
    f32_a = torch.empty(n, 3, h, w, device="cuda")
    f32_b = torch.full((n, 3, h, w), float("nan"), device="cuda")
    u8_a = eng.enhance(frames, mode=mode, out_f32=f32_a)
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    u8_b = eng.enhance_tiled(frames, tile=tile, mode=mode, out_f32=f32_b, max_pass_pixels=max_pass_pixels)
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    if not torch.equal(u8_a, u8_b):
        pytest.fail("out_u8: " + _where((u8_a != u8_b).any(-1).cpu().numpy(), h, w, tile))
    if not torch.equal(f32_a, f32_b):
        pytest.fail("out_f32: " + _where((f32_a != f32_b).any(1).cpu().numpy(), h, w, tile))
    return u8_b, f32_b


@pytest.mark.parametrize("precision", ["bf16x3", "bf16_fp8"])
def test_tiled_equals_untiled_over_several_passes(precision):
    """3 x 300x520 frames, tile 64x96: 90 windows of 113x86, 40 per pass -> passes of 40, 40 and 10."""
    from waternet_b200.engine import tile_geometry
    m = _model(ofw.synthetic_state_dict(0, 3.0), precision)
    g = tile_geometry(300, 520, 64, 96)
    assert (g["win_h"], g["win_w"], len(g["windows"])) == (86, 113, 30)
    _assert_same(m.engine(), _frames(3, 300, 520), MODE[precision], (64, 96),
                 max_pass_pixels=40 * g["win_h"] * g["win_w"] + 5)


@pytest.mark.parametrize("h,w,tile", [
    (37, 53, (256, 256)),    # the image is smaller than one window
    (40, 700, (128, 128)),   # one axis smaller than the window
    (113, 117, (32, 32)),    # sizes that are not multiples of 8
    (192, 256, (64, 128)),   # the tile divides the image exactly
    (50, 70, (8, 8)),        # tile 8: windows of 34 x 34
])
def test_tiled_equals_untiled_edge_shapes(h, w, tile):
    m = _model(ofw.synthetic_state_dict(3, 3.0))
    _assert_same(m.engine(), _frames(2, h, w, seed=10), MODE["default"], tile)


@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
def test_tiled_equals_untiled_full_size_frames(h, w):
    m = _model(ofw.synthetic_state_dict(0, 3.0))
    eng = m.engine()
    try:
        _assert_same(eng, _frames(1, h, w, seed=40), MODE["default"], eng.DEFAULT_TILE)
    finally:
        eng.release_workspaces()


def test_8k_frame_tiled_against_the_oracle_on_crops():
    """One 7680x4320 frame (untiled: 62 GB of workspace).  out_f32 on crops at the corners, the borders, tile seams
    and the interior against the CPU oracle, each crop run with 13 pixels of context (cut at the image borders)."""
    from waternet_b200.engine import TILE_HALO, tile_geometry
    h, w = 4320, 7680
    sd = ofw.synthetic_state_dict(0, 3.0)
    m = _model(sd)
    eng = m.engine()
    need = eng.tiled_workspace_bytes(1, h, w)
    g = tile_geometry(h, w, *eng.DEFAULT_TILE)
    assert need < 16e9 and need >= 9 * g["win_h"] * g["win_w"] * 1868
    assert eng.lib.wn_enhance_workspace_bytes(1, h, w, -1) > 60e9
    rgb = _frames(1, h, w, seed=50)
    f32 = torch.empty(1, 3, h, w, device="cuda")
    try:
        u8 = eng.enhance_tiled(rgb, out_f32=f32).cpu().numpy()
        pre = eng.preprocess(rgb)
        ins = [pre[k].cpu() for k in ("x", "wb", "he", "gc")]
    finally:
        eng.release_workspaces()
    assert not eng.f8_overflowed()
    out = f32.cpu().numpy()
    sy, sx = 2 * g["th"], 4 * g["tw"]  # a seam row / column
    s = 24
    crops = [(0, 0), (0, w - s), (h - s, 0), (h - s, w - s),      # corners
             (0, sx - s // 2), (sy - s // 2, 0),                    # borders across a seam
             (h - s, sx - s // 2), (sy - s // 2, w - s),
             (sy - s // 2, sx - s // 2),                            # a seam crossing (seam +-1 inside)
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


def test_range_guard_rerun_on_the_tiled_path():
    """Weights whose activations leave the e4m3 range on the first pass: the default mode recomputes every pass
    with the bf16x3 kernels, so its output equals the bf16x3 output bit for bit."""
    sd = ofw.synthetic_state_dict(0, 3.0)
    sd["wb_refiner.conv1.weight"] = sd["wb_refiner.conv1.weight"] * 400.0
    sd["wb_refiner.conv2.weight"] = sd["wb_refiner.conv2.weight"] / 400.0
    frames = _frames(2, 120, 200, seed=30)
    f8, plain = _model(sd, "default"), _model(sd, "bf16x3")
    f32_a, f32_b = torch.empty(2, 3, 120, 200, device="cuda"), torch.empty(2, 3, 120, 200, device="cuda")
    a = f8.engine().enhance_tiled(frames, tile=48, mode=MODE["default"], out_f32=f32_a, max_pass_pixels=10000)
    b = plain.engine().enhance_tiled(frames, tile=48, mode=MODE["bf16x3"], out_f32=f32_b, max_pass_pixels=10000)
    torch.cuda.synchronize()
    assert f8.engine().f8_overflowed()
    assert torch.equal(a, b) and torch.equal(f32_a, f32_b)


def test_enhancer_with_tile_equals_whole_image_enhancer():
    from waternet_b200.api import Enhancer
    m = _model(ofw.synthetic_state_dict(0, 3.0))
    whole, tiled = Enhancer(m), Enhancer(m, tile=(64, 96))
    batch = _frames(3, 300, 520, seed=60).cpu().numpy()
    want = whole(batch)
    assert np.array_equal(tiled(batch), want)
    assert np.array_equal(tiled(batch[1]), want[1])
    batches = [_frames(2, 300, 520, seed=70 + 5 * k).cpu().numpy() for k in range(5)]
    wants = [whole(b) for b in batches]
    pins = [(torch.from_numpy(b).pin_memory(), torch.empty(b.shape, dtype=torch.uint8).pin_memory()) for b in batches]
    deep = Enhancer(m, tile=(64, 96), depth=3)
    tickets = [deep.submit(*pins[k]) for k in range(3)]   # three batches in flight
    for k in range(3, 5):
        deep.wait(tickets[k - 3])
        tickets.append(deep.submit(*pins[k]))
    for t in tickets:
        deep.wait(t)
    for (_, po), ref in zip(pins, wants):
        assert np.array_equal(po.numpy(), ref)
    assert all(slot.graph is None for slot in tiled._slots + deep._slots)


def test_enhancer_tile_rejects_what_it_cannot_do():
    from waternet_b200.api import Enhancer
    m = _model(ofw.synthetic_state_dict(0, 1.0))
    with pytest.raises(ValueError):
        Enhancer(m, precision="fp32", tile=64)
    with pytest.raises(ValueError):
        Enhancer(m, tile=0)
    enh = Enhancer(m, tile=64)
    pin = torch.empty(1, 32, 32, 3, dtype=torch.uint8).pin_memory()
    with pytest.raises(ValueError):
        enh.submit(pin, torch.empty_like(pin).pin_memory(), exchange=object())
    from waternet_b200 import _lib
    with pytest.raises(_lib.WaterNetLibraryError, match="FP32"):
        m.engine().enhance_tiled(_frames(1, 32, 32), tile=16, mode=_lib.MODE_FP32_SIMT)
