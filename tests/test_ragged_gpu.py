"""Ragged batches (wn_enhance_u8_ragged) on the GPU: each image's outputs bit-identical to enhancing it alone."""
import numpy as np
import pytest
import torch

from oracle import forward as ofw

pytestmark = pytest.mark.gpu

MODE = {"bf16x3": 1, "bf16_fp8": 2, "default": -1}
SIZES = [(5, 7), (37, 53), (113, 117), (112, 112), (300, 520), (40, 700), (1080, 1920)]
TILE = (256, 256)
SMALL_PASS = 200_000  # several passes, some mixing window sizes


def _model(sd, precision="default"):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _images(sizes, seed=0):
    return [torch.from_numpy(ofw.synthetic_image(seed + i, h, w, "smooth" if i % 2 else "noise")).cuda()
            for i, (h, w) in enumerate(sizes)]


def _where(diff, h, w, tile):
    """Where an (H, W) mismatch mask of one image lies: at the bottom / right border, where the masked padding of a
    slot begins (a masking bug); at the seams between kept rectangles (a geometry bug); or in the interior."""
    from waternet_b200.engine import tile_geometry
    g = tile_geometry(h, w, *tile)
    seams_y = np.array([k0 for _, _, (k0, _), _ in g["windows"] if k0 > 0] or [-99])
    seams_x = np.array([k0 for _, _, _, (k0, _) in g["windows"] if k0 > 0] or [-99])
    idx = np.argwhere(diff)
    edge = (idx[:, 0] >= h - 3) | (idx[:, 1] >= w - 3)
    seam = ~edge & ((np.abs(idx[:, 0, None] - seams_y[None]).min(1) <= 2)
                    | (np.abs(idx[:, 1, None] - seams_x[None]).min(1) <= 2))
    return (f"{len(idx)} pixels differ: {int(edge.sum())} at the mask edge, {int(seam.sum())} at window seams, "
            f"{int((~edge & ~seam).sum())} in the interior; first (y, x): {tuple(idx[0])}")


def _alone(eng, images, mode):
    """enhance of each image alone: uint8 and fp32 outputs; the range flag stays down."""
    u8, f32 = [], []
    for img in images:
        h, w, _ = img.shape
        f = torch.empty(1, 3, h, w, device="cuda")
        u8.append(eng.enhance(img[None], mode=mode, out_f32=f)[0])
        f32.append(f)
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    return u8, f32


def _ragged(eng, images, mode, tile=TILE, max_pass_pixels=SMALL_PASS):
    f32 = [torch.full((1, 3, img.shape[0], img.shape[1]), float("nan"), device="cuda") for img in images]
    u8 = eng.enhance_ragged(images, tile=tile, mode=mode, out_f32=f32, max_pass_pixels=max_pass_pixels)
    torch.cuda.synchronize()
    return u8, f32


def _assert_same(want, got, tile=TILE):
    (wu, wf), (gu, gf) = want, got
    for i, (a, b) in enumerate(zip(wu, gu)):
        h, w, _ = a.shape
        if not torch.equal(a, b):
            pytest.fail(f"image {i} ({h}x{w}) out_u8: " + _where((a != b).any(-1).cpu().numpy(), h, w, tile))
        if not torch.equal(wf[i], gf[i]):
            pytest.fail(f"image {i} ({h}x{w}) out_f32: " + _where((wf[i] != gf[i]).any(1)[0].cpu().numpy(), h, w, tile))


def test_plan_of_the_test_mix_masks():
    from waternet_b200.engine import ragged_plan
    passes = ragged_plan(SIZES, *TILE, SMALL_PASS)
    assert len(passes) > 2
    assert any(len({(r["vh"], r["vw"]) for r in p["windows"]}) > 1 for p in passes)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16_fp8"])
def test_ragged_equals_each_image_alone(precision):
    m = _model(ofw.synthetic_state_dict(0, 3.0), precision)
    eng = m.engine()
    images = _images(SIZES)
    want = _alone(eng, images, MODE[precision])
    got = _ragged(eng, images, MODE[precision])
    assert not eng.f8_overflowed()
    _assert_same(want, got)


def test_stale_workspace_does_not_leak_into_the_result():
    """The workspace starts as 0xFF bytes (bf16 NaN): a slot pixel that is not stored as zero would show in the
    output, and in the fp8-correction mode it would raise the e4m3 flag."""
    m = _model(ofw.synthetic_state_dict(1, 3.0))
    eng = m.engine()
    images = _images(SIZES, seed=20)
    want = _alone(eng, images, MODE["default"])
    nbytes = eng.ragged_workspace_bytes([tuple(i.shape[:2]) for i in images], TILE, MODE["default"], SMALL_PASS)
    eng._workspace("enhance", nbytes).fill_(0xFF)
    got = _ragged(eng, images, MODE["default"])
    assert not eng.f8_overflowed()
    _assert_same(want, got)


def test_one_image_equals_the_tiled_call():
    m = _model(ofw.synthetic_state_dict(2, 3.0))
    eng = m.engine()
    img = _images([(300, 520)], seed=30)[0]
    f_t = torch.empty(1, 3, 300, 520, device="cuda")
    tiled = eng.enhance_tiled(img[None], tile=(64, 96), out_f32=f_t, max_pass_pixels=40_000)[0]
    u8, f32 = _ragged(eng, [img], MODE["default"], tile=(64, 96), max_pass_pixels=40_000)
    assert torch.equal(tiled, u8[0]) and torch.equal(f_t, f32[0])


def test_equally_sized_images_equal_the_stacked_batch():
    m = _model(ofw.synthetic_state_dict(0, 3.0))
    eng = m.engine()
    images = _images([(120, 200)] * 4, seed=40)
    f_b = torch.empty(4, 3, 120, 200, device="cuda")
    batch = eng.enhance(torch.stack(images), out_f32=f_b)
    u8, f32 = _ragged(eng, images, MODE["default"], max_pass_pixels=0)
    for i in range(4):
        assert torch.equal(batch[i], u8[i]) and torch.equal(f_b[i:i + 1], f32[i])


def test_zero_pixel_images_get_empty_outputs():
    m = _model(ofw.synthetic_state_dict(0, 3.0))
    eng = m.engine()
    empty = [torch.empty(0, 5, 3, dtype=torch.uint8, device="cuda"), torch.empty(4, 0, 3, dtype=torch.uint8,
                                                                                   device="cuda")]
    img = _images([(37, 53)], seed=45)[0]
    out = eng.enhance_ragged([empty[0], img, empty[1]])
    assert [tuple(o.shape) for o in out] == [(0, 5, 3), (37, 53, 3), (4, 0, 3)]
    assert torch.equal(out[1], eng.enhance(img[None])[0])
    before = eng.launch_count
    assert [tuple(o.shape) for o in eng.enhance_ragged(empty)] == [(0, 5, 3), (4, 0, 3)]
    assert eng.launch_count == before  # no library call


def test_range_guard_rerun_on_the_ragged_path():
    """Weights whose activations leave the e4m3 range: the default mode recomputes the passes with the bf16x3
    kernels, so its output equals the bf16x3 ragged output and each image's bf16x3 enhance, bit for bit."""
    sd = ofw.synthetic_state_dict(0, 3.0)
    sd["wb_refiner.conv1.weight"] = sd["wb_refiner.conv1.weight"] * 400.0
    sd["wb_refiner.conv2.weight"] = sd["wb_refiner.conv2.weight"] / 400.0
    images = _images(SIZES[:6], seed=50)
    f8, plain = _model(sd, "default"), _model(sd, "bf16x3")
    got = _ragged(f8.engine(), images, MODE["default"])
    assert f8.engine().f8_overflowed()
    want = _ragged(plain.engine(), images, MODE["bf16x3"])
    _assert_same(want, got)
    _assert_same(_alone(plain.engine(), images, MODE["bf16x3"]), got)


def test_enhancer_enhance_many():
    from waternet_b200.api import Enhancer
    m = _model(ofw.synthetic_state_dict(0, 3.0))
    arrs = [i.cpu().numpy() for i in _images(SIZES[:6], seed=60)]
    want = [Enhancer(m)(a) for a in arrs]
    for enh in (Enhancer(m), Enhancer(m, tile=64)):
        got = enh.enhance_many(arrs)
        assert len(got) == len(arrs)
        for a, b in zip(want, got):
            assert a.shape == b.shape and np.array_equal(a, b)
        assert all(np.array_equal(a, b) for a, b in zip(want[:2], enh.enhance_many(arrs[:2])))  # staging reused
    with pytest.raises(ValueError):
        Enhancer(m, precision="fp32").enhance_many(arrs)
