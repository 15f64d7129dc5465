"""The first launch's fp8 tap-pair form on the GPU (DESIGN section 4.2; emulated in test_first_layer_f8_cpu.py).

In the fp8-correction mode, level inputs run L1 (layers 0 and 8) as 25 e4m3 wgmmas over tap pairs plus 49 bf16
wgmmas, and float inputs run its bf16x3 form in the same launch.  The per-launch check compares layers 0 and 8 with
float64 through ``debug_layer`` at the bf16_fp8 bar, with no fp8 floor beyond the one of the stored output.
"""
import pytest
import torch

import forward_reference as fr
from test_conv_tiles_gpu import SHAPES

pytestmark = pytest.mark.gpu

MODE = "bf16_fp8"


def _model(sd, precision=MODE):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _check_first_layer(m, sd, ins, label):
    eng = m.engine()
    cu = [t.cuda() for t in ins]
    worst = 0.0
    for layer in (0, 8):
        G = eng.debug_layer(*cu, layer=layer, mode=m._mode())
        assert torch.isfinite(G).all(), (label, layer)
        ref = fr.layer_reference(sd, layer, cu, MODE)
        fr.check(G, ref, fr.TAU[MODE], f"{label} {fr.LAYER_NAMES[layer]}")
        worst = max(worst, fr.excess(G, ref))
    return worst


def test_tap_pairs_at_one_small_shape():
    """One tile: a descriptor LBO of 16 B (two taps one pixel apart) addresses the second core matrix as computed."""
    sd = fr.weight_set("stress", 3)
    _check_first_layer(_model(sd), sd, fr.make_inputs("levels", 1, 16, 8, 7), "1 x 16 x 8")


@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
def test_first_layer_at_tile_edges(weights):
    sd = fr.weight_set(weights, 4)
    m = _model(sd)
    worst = 0.0
    for i, kind in enumerate(("levels", "dark_levels")):
        for n, h, w in SHAPES + [(2, 37, 53)]:
            worst = max(worst, _check_first_layer(m, sd, fr.make_inputs(kind, n, h, w, 100 * i + h * 7 + w),
                                                  f"{weights} {kind} {(n, h, w)}"))
    print(f"{weights}: worst (|G - R| - F) / M of layers 0 and 8: {worst:.2e}")


@pytest.mark.parametrize("layer", [0, 8])
def test_float_inputs_keep_the_bf16x3_form(layer):
    """Float inputs run the bf16x3 form: the default-mode output equals the bf16x3-mode one up to the storage of the
    correction in e4m3 (2^-13 relative to the value, 2^-19 absolute).  The tap-pair form would drop a_lo x w_hi, a
    2^-9 relative error."""
    sd = fr.weight_set("stress", 5)
    ins = [t.cuda() for t in fr.make_inputs("floats", 2, 37, 53, 9)]
    m8, m3 = _model(sd), _model(sd, "bf16x3")
    e = m8.engine().debug_layer(*ins, layer=layer, mode=m8._mode()).double()
    d = m3.engine().debug_layer(*ins, layer=layer, mode=m3._mode()).double()
    assert ((e - d).abs() <= 2.0 ** -13 * d.abs() + 2.0 ** -19).all(), (e - d).abs().max().item()
    assert (e != d).any()  # two storage formats: the default mode really ran with its own epilogue
