"""The first launch's fp8 tap-pair form (DESIGN section 4.2), emulated in float64 against the per-launch bar.

For 8-bit-level inputs the fp8-correction mode computes L1 (cmg.conv1 and the three refiner conv1, layers 0 and 8) as
    acc = sum_pairs e4m3(a) x e4m3(w_lo s_c 2^9)      (25 e4m3 wgmmas of K = 32: two taps of 16 channels each)
    acc += sum_taps a x bf16(w) s_c 2^9               (49 bf16 wgmmas of K = 16; a level is exact in bf16)
    v = acc 2^-9 / s_c + b
with s_c a power of two per output column (max|w| of the column in [112, 224]).  The fp8 products are issued first,
so the accumulator holds only correction sums while Hopper's fp8 MMA adds into it.  The emulation takes every product
exactly, walks the kernel's pair table (``PAIRS``) and stores the result as L1 stores it (hi + fp8 planes).  It must
pass the bf16_fp8 bar of layers 0 and 8, which have no fp8 floor beyond the WRITES_F8 one; each fault must fail it.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import forward_reference as fr

KS = 7
HALO_W, HALO_H = 8 + KS - 1, 16 + KS - 1   # the halo tile of an 8 x 16-pixel tile, two consumer warpgroups
SHAPES = [(1, 19, 24), (2, 37, 53)]


def pairs(kk=KS * KS):
    """The kernel's pair table (conv_umma_kernel, kFmtPair8): pair p multiplies the fp8 plane at taps t0 and t0 + 1
    (one descriptor: start at tap t0, LBO = the distance to tap t0 + 1).  The odd last tap is paired with a
    zero-weight partner below it, so that no read leaves the halo plane.  (t0, t1, t0 carries weights)."""
    return [(min(2 * p, kk - 2), min(2 * p, kk - 2) + 1, 2 * p < kk - 1) for p in range((kk + 1) // 2)]


PAIRS = pairs()


def column_scales(w):
    """s_c of pair_scale_kernel: 2^floor(log2(224 / max|w|)) over each output column, in fp32."""
    mx = np.maximum(w.abs().amax(dim=(1, 2, 3)).float().numpy(), np.float32(1e-30))
    return torch.from_numpy(np.exp2(np.floor(np.log2(np.float32(224.0) / mx))).astype(np.float64))


def _tap(x, wt, dy, dx):
    """sum_c wt[o, c] x[c, y + dy - 3, x + dx - 3] (zero outside the image): one tap read at offset (dy, dx)."""
    n, c, h, w = x.shape
    xp = F.pad(x, (KS // 2, KS // 2 + 2, KS // 2, KS // 2))
    return F.conv2d(xp[:, :, dy:dy + h, dx:dx + w], wt[:, :, None, None])


def emulate_pair_form(sd, layer, images, fault=None):
    """Layer 0 or 8 in the fp8 tap-pair form, from four level images; returns the decoded stored output."""
    ops, exact = fr._first_operands(images)
    assert exact, "the tap-pair form runs on 8-bit-level inputs only"
    a8 = fr._e4m3(ops)
    zs = []
    blocks = fr._blocks(layer)
    ws_layer = fr.f8_ws({p + ".weight": sd[p + ".weight"] / 255 for p, _, _, _ in blocks}, layer)
    for prefix, k, src, _ in blocks:
        assert k == KS
        w = fr._f32(sd[prefix + ".weight"].double() / 255)
        b = sd[prefix + ".bias"].double()
        cols = slice(None) if src[1] is None else [0, 1, 2, 3 * (src[1] + 1), 3 * (src[1] + 1) + 1, 3 * (src[1] + 1) + 2]
        x, x8 = ops[:, cols], a8[:, cols]
        s = column_scales(w)
        if fault == "layer_scale":
            s = torch.full_like(s, ws_layer)
        sv = s.view(-1, 1, 1, 1)
        w_hi = fr._bf16(w)
        q = fr._e4m3(fr._f32(w - w_hi) * sv * 512)
        main = F.conv2d(x, w_hi * sv * 512, None, padding=KS // 2)
        corr = torch.zeros_like(main)
        for p, (t0, t1, weighted) in enumerate(PAIRS):
            reads = [(t0, t0 if weighted else None), (t1, t1)]
            for pos, wt in reads:
                if wt is None:
                    continue
                dy, dx = divmod(pos, KS)
                if fault == "pair_offset" and pos == t1:
                    dx += 1   # every second K half one pixel further along the halo row (LBO off by 16 B)
                corr = corr + _tap(x8, q[:, :, wt // KS, wt % KS], dy, dx)
        if fault == "drop_correction":
            corr = 0 * corr
        if fault == "correction_2x":
            corr = 2 * corr
        z = fr._f32(fr._f32(corr + main) * (2.0 ** -9 / sv.view(1, -1, 1, 1)))
        zs.append(fr._f32(z + b.view(1, -1, 1, 1)))
    v = F.relu(torch.cat(zs, 1))
    return fr._store(v, "f8").value


def _worst(sd, ins, fault=None):
    return max(fr.excess(emulate_pair_form(sd, layer, ins, fault), fr.layer_reference(sd, layer, ins, "bf16_fp8"))
               for layer in (0, 8))


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(8, n))
    yield
    torch.set_num_threads(n)


def test_pair_table_covers_every_tap_once_inside_the_halo():
    weighted = [t for t0, t1, w0 in PAIRS for t in ((t0, t1) if w0 else (t1,))]
    assert sorted(weighted) == list(range(KS * KS))
    assert len(PAIRS) == 25
    # every byte a pair's two K halves read, for the 64 rows of either warpgroup (8 halo rows of 8 pixels from row
    # 8 wg on), lies inside that warpgroup's 14 halo rows of the plane
    for t0, t1, _ in PAIRS:
        off0 = ((t0 // KS) * HALO_W + t0 % KS) * 16
        lbo = ((t1 // KS) * HALO_W + t1 % KS) * 16 - off0
        assert 0 < lbo < (1 << 18) and lbo % 16 == 0
        for wg in range(2):
            base = wg * 8 * HALO_W * 16
            lo = base + off0
            hi = base + off0 + lbo + 7 * HALO_W * 16 + 7 * 16 + 16
            assert lo >= wg * 8 * HALO_W * 16 and hi <= (wg * 8 + KS + 7) * HALO_W * 16, (t0, t1, wg)
            assert hi <= HALO_W * HALO_H * 16


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
def test_emulated_pair_form_passes_the_bar(weights, shape):
    sd = fr.weight_set(weights, 1)
    worst = 0.0
    for i, kind in enumerate(("levels", "dark_levels")):
        ins = fr.make_inputs(kind, *shape, 50 + i)
        for layer in (0, 8):
            ref = fr.layer_reference(sd, layer, ins, "bf16_fp8")
            G = emulate_pair_form(sd, layer, ins)
            fr.check(G, ref, fr.TAU["bf16_fp8"], f"{weights} {kind} {fr.LAYER_NAMES[layer]}")
            worst = max(worst, fr.excess(G, ref))
    print(f"{weights} {shape}: worst excess {worst:.3e}")
    assert worst < fr.TAU["bf16_fp8"] / 2


def test_column_scales_beat_one_scale_per_launch():
    """One scale per launch puts the graded weights' small columns into e4m3's subnormals.  The bar cannot tell (a
    subnormal w_lo operand costs about 2^-19 of a product, and columns small enough to lose more sit under the 2^-19
    storage floor), so this compares the worst excess itself: the per-column scales keep it lower."""
    sd = fr.weight_set("graded", 1)
    ins = fr.make_inputs("levels", *SHAPES[0], 61)
    err = lambda fault: max((emulate_pair_form(sd, layer, ins, fault) - fr.layer_reference(sd, layer, ins).R).abs()
                            .div(fr.layer_reference(sd, layer, ins).M.clamp_min(1e-30)).max().item() for layer in (0, 8))
    assert err(None) <= err("layer_scale")


@pytest.mark.parametrize("fault", ["pair_offset", "drop_correction", "correction_2x"])
def test_fault_fails_the_bar(fault):
    sd = fr.weight_set("stress", 1)
    ins = fr.make_inputs("levels", *SHAPES[0], 60)
    assert _worst(sd, ins) < fr.TAU["bf16_fp8"]
    assert _worst(sd, ins, fault) > fr.TAU["bf16_fp8"], fault
