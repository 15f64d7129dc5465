"""The 16 x 16-pixel tiles of the tensor-core convolutions at the shapes they add: the ragged and tiled enhance paths
with window extents that are not multiples of 16.  SHAPES -- widths of 8 (mod 16), where a whole m64 block of a tile
lies outside the image; every height (mod 16); 1 x 1 and 16 x 8 images -- is where test_forward_layers_gpu.py checks
every launch against float64."""
import pytest
import torch

from oracle import forward as ofw

pytestmark = pytest.mark.gpu

TC_MODES = ["bf16x3", "bf16_fp8"]
# (n, h, w): widths 8, 24, 40 and 56 are 8 (mod 16); the heights cover 1..15 (mod 16)
SHAPES = [(1, 1, 1), (1, 16, 8), (2, 17, 24), (1, 18, 40), (1, 19, 8), (1, 20, 56), (1, 21, 23), (1, 22, 72),
          (1, 23, 9), (1, 24, 40), (1, 25, 31), (1, 26, 24), (1, 27, 88), (1, 28, 17), (1, 29, 104), (1, 30, 8),
          (1, 31, 120), (3, 47, 61)]


def _model(precision):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(ofw.synthetic_state_dict(11, 3.0), strict=True)
    return m.cuda().eval()


def _frames(sizes, seed):
    return [torch.from_numpy(ofw.synthetic_image(seed + i, h, w, "smooth" if i % 2 else "noise")).cuda()
            for i, (h, w) in enumerate(sizes)]


@pytest.mark.parametrize("precision", TC_MODES)
def test_tiled_enhance_bitwise_with_ragged_windows(precision):
    """enhance_tiled with windows whose extents are not multiples of 16 gives the untiled call's bits."""
    m = _model(precision)
    eng = m.engine()
    mode = m._mode()
    for (h, w), tile in [((120, 200), (37, 53)), ((93, 141), (45, 29)), ((64, 72), (21, 40))]:
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
def test_ragged_enhance_bitwise_at_tile_edges(precision):
    """A ragged call over images whose sizes and windows are not multiples of 16 gives each image's bits alone."""
    m = _model(precision)
    eng = m.engine()
    mode = m._mode()
    sizes = [(1, 1), (16, 8), (17, 24), (29, 40), (37, 53), (70, 90), (113, 117)]
    images = _frames(sizes, 40)
    want_u8, want_f32 = [], []
    for img in images:
        f = torch.empty(1, 3, img.shape[0], img.shape[1], device="cuda")
        want_u8.append(eng.enhance(img[None], mode=mode, out_f32=f)[0])
        want_f32.append(f)
    got_f32 = [torch.full_like(f, float("nan")) for f in want_f32]
    got_u8 = eng.enhance_ragged(images, tile=(45, 61), mode=mode, out_f32=got_f32, max_pass_pixels=30_000)
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    for i, (h, w) in enumerate(sizes):
        assert torch.equal(want_u8[i], got_u8[i]), (h, w)
        assert torch.equal(want_f32[i], got_f32[i]), (h, w)
