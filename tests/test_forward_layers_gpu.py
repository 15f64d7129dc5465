"""Every launch of the forward pass, in each precision, element by element against float64 on the launch's own input.

For each mode (fp32 CUDA-core, bf16x3, bf16_fp8) the ten launches (eleven outputs: the first launch has two) are read
back through ``wn_debug_forward_layer`` and each is checked with ``forward_reference``: |G - R| <= tau M + F, R and M
computed in float64 on the device from the decoded input the launch consumed.  Then the gated output: ``m(*ins)``
must equal sum_r refined_r cm_r of the maps (layer 7) and refined images (layer 10) within the same bar, which ties
the debug chain to the real forward.  Shapes: 1 x 1, widths of 8 (mod 16), every height (mod 16), a batch of 3,
2 x 37 x 53 and 1 x 300 x 500 (many tiles per CTA).  Inputs: 8-bit levels (the first launch's 2-pass form), floats
(3-pass), dark floats in [0, 0.02] and level images with a near-black region.  Weights: stress (gain 3), default
init, the 400-epoch trained set and the graded set (forward_reference.graded_state_dict).
"""
import pytest
import torch

import forward_reference as fr
from test_conv_tiles_gpu import SHAPES

pytestmark = pytest.mark.gpu

EDGE_SHAPES = SHAPES + [(2, 37, 53), (1, 300, 500)]


def _model(sd, precision):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _check_case(m, sd, mode, ins, worst, label, forward=True):
    """Every launch of one forward and the gated output; worst[(layer)] keeps the largest excess (|G - R| - F) / M.
    forward=False: the launches alone, for weights on which the forward is expected to raise the range flag."""
    eng = m.engine()
    tau = fr.TAU[mode]
    cu = [t.cuda() for t in ins]
    outs = {}
    for layer in range(11):
        G = eng.debug_layer(*cu, layer=layer, mode=m._mode())
        assert G.shape == (ins[0].shape[0], fr.CHANNELS[layer]) + tuple(ins[0].shape[2:])
        assert torch.isfinite(G).all(), (label, layer)
        src = cu if fr.INPUT_LAYER[layer] is None else outs[fr.INPUT_LAYER[layer]]
        ref = fr.layer_reference(sd, layer, src, mode)
        fr.check(G, ref, tau, f"{label} {mode} {fr.LAYER_NAMES[layer]}")
        worst[layer] = max(worst.get(layer, 0.0), fr.excess(G, ref))
        outs[layer] = G
    if not forward:
        return
    with torch.no_grad():
        out = m(*cu)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all(), label
    assert not eng.f8_overflowed(), label
    gate = fr.gate_reference(outs[fr.MAPS], outs[fr.REFINED])
    fr.check(out, gate, tau, f"{label} {mode} gated output")
    worst["gate"] = max(worst.get("gate", 0.0), fr.excess(out, gate))


def _report(title, worst):
    print(f"{title}: worst (|G - R| - F) / M per launch: " +
          " ".join(f"{fr.LAYER_NAMES[k].split(' ')[0] if k != 'gate' else 'gate'}={v:.2e}" for k, v in worst.items()))


@pytest.mark.parametrize("mode", fr.MODES)
def test_every_launch_at_tile_edges(mode):
    """Stress weights, random floats, at every shape of EDGE_SHAPES."""
    sd = fr.weight_set("stress", 11)
    m = _model(sd, mode)
    worst = {}
    for n, h, w in EDGE_SHAPES:
        _check_case(m, sd, mode, fr.make_inputs("floats", n, h, w, h * 1000 + w), worst, f"{(n, h, w)}")
    _report(f"{mode} shapes", worst)


@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
@pytest.mark.parametrize("mode", fr.MODES)
def test_every_launch_per_weight_set_and_input(mode, weights):
    """Each weight set with level, float, dark-float and dark-level inputs, at 2 x 37 x 53."""
    sd = fr.weight_set(weights, 2)
    m = _model(sd, mode)
    worst = {}
    for i, kind in enumerate(fr.INPUT_KINDS):
        _check_case(m, sd, mode, fr.make_inputs(kind, 2, 37, 53, 50 + i), worst, f"{weights} {kind}")
    _report(f"{mode} {weights}", worst)


def test_cpu_and_cuda_references_agree():
    """The float64 reference (R, M and the fp8 floor) does not depend on the device it runs on."""
    sd = fr.weight_set("graded", 3)
    ins = fr.make_inputs("floats", 1, 13, 21, 9)
    torch.manual_seed(0)
    for layer in range(11):
        a = ins if fr.INPUT_LAYER[layer] is None else torch.rand(1, fr.CHANNELS[fr.INPUT_LAYER[layer]], 13, 21)
        cpu = fr.layer_reference(sd, layer, a, "bf16_fp8")
        gpu = fr.layer_reference(sd, layer, [t.cuda() for t in a] if isinstance(a, list) else a.cuda(), "bf16_fp8")
        # each device's float64 summation order (and exp) shows relative to the magnitudes M + F / tau, not to R
        tau = fr.TAU["bf16_fp8"]
        bar = cpu.M + cpu.F / tau
        assert ((gpu.R.cpu() - cpu.R).abs() <= 1e-11 * bar).all(), layer
        assert ((gpu.M.cpu() + gpu.F.cpu() / tau - bar).abs() <= 1e-11 * bar).all(), layer
