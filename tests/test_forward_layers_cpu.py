"""The per-launch forward check of test_forward_layers_gpu.py tells the documented arithmetic from weaker ones.

forward_reference.emulate_layer restates each mode's operand formats with exact float64 products.  Its results must
pass the committed bar at every launch (else tau was fitted to luck); the fp8 floor must be what lets the bf16_fp8
results pass on the graded and trained weights (else it would be slack that hides a bug); and each fault of
forward_reference.FAULTS -- a dropped bf16x3 correction term, an fp8 scale off by 2x, a shifted tap, swapped channels,
a zeroed edge row or column, one channel at bf16-only precision, TF32 weights in the fp32 mode -- must fail it.
"""
import pytest
import torch

import forward_reference as fr

SHAPE = (1, 19, 24)  # one full 16 x 16 tile and partial ones on both axes


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(8, n))
    yield
    torch.set_num_threads(n)


def _chain(sd, ins, mode, fault=None, fault_layer=None):
    acts = {}
    for layer in range(11):
        src = ins if fr.INPUT_LAYER[layer] is None else acts[fr.INPUT_LAYER[layer]]
        acts[layer] = fr.emulate_layer(sd, layer, src, mode, fault if layer == fault_layer else None)
    return acts


def _layer_input(ins, acts, layer):
    return ins if fr.INPUT_LAYER[layer] is None else acts[fr.INPUT_LAYER[layer]].value


@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
@pytest.mark.parametrize("mode", fr.MODES)
def test_emulated_arithmetic_passes_the_bar(mode, weights):
    """Every launch and the gated output of the emulated mode, for every input kind, at the committed tau."""
    sd = fr.weight_set(weights, 1)
    for i, kind in enumerate(fr.INPUT_KINDS):
        ins = fr.make_inputs(kind, *SHAPE, 20 + i)
        acts = _chain(sd, ins, mode)
        for layer in range(11):
            ref = fr.layer_reference(sd, layer, _layer_input(ins, acts, layer), mode)
            fr.check(acts[layer].value, ref, fr.TAU[mode], f"{weights} {kind} {mode} {fr.LAYER_NAMES[layer]}")
        maps, refined = acts[fr.MAPS].value, acts[fr.REFINED].value
        fr.check(fr.emulate_gate(maps, refined), fr.gate_reference(maps, refined), fr.TAU[mode], "gated output")


@pytest.mark.parametrize("weights,kind", [("graded", "floats"), ("graded", "dark_floats"), ("trained", "floats")])
def test_fp8_floor_is_a_property_of_the_format(weights, kind):
    """Without the floor the emulated bf16_fp8 results fail the bar on the graded weights (activations and weights in
    e4m3's subnormal range) and on the trained weights (cmg.conv2 has weights below 2^-6 / ws); with it they pass
    (test above).  Dark inputs alone do not need it: their activations stay above the subnormal range after the
    first launch's bias."""
    sd = fr.weight_set(weights, 1)
    ins = fr.make_inputs(kind, *SHAPE, 30)
    acts = _chain(sd, ins, "bf16_fp8")
    worst = max(fr.excess(acts[layer].value, fr.layer_reference(sd, layer, _layer_input(ins, acts, layer)))
                for layer in range(11))
    assert worst > fr.TAU["bf16_fp8"], worst


# (fault, mode, launch): the launch that computes wrongly
REJECTED = [
    ("drop_w_lo", "bf16x3", 6),               # cmg.conv7 without a_hi x w_lo
    ("drop_w_lo_second_block", "bf16x3", 4),  # cmg.conv5, one 16 x 16 tile's second m64 block only
    ("drop_w_lo_second_block", "bf16x3", 6),
    ("skip_lo", "bf16x3", 0),                 # the first launch drops a_lo on float inputs
    ("skip_lo", "bf16_fp8", 8),
    ("f8_scale_2x", "bf16_fp8", 4),           # dequantisation scale 2^-8 / ws instead of 2^-9 / ws
    ("f8_scale_2x", "bf16_fp8", 9),
    ("shifted_tap", "bf16x3", 5),
    ("swapped_channels", "bf16x3", 2),
    ("swapped_channels", "fp32", 10),
    ("zero_edge_row", "bf16_fp8", 3),
    ("zero_edge_column", "bf16x3", 9),
    ("bf16_channel", "bf16x3", 1),
    ("bf16_channel", "bf16x3", 3),
    ("tf32_weights", "fp32", 0),
    ("tf32_weights", "fp32", 3),
    ("tf32_weights", "fp32", 6),
]


@pytest.mark.parametrize("fault,mode,layer", REJECTED)
def test_check_rejects_fault(fault, mode, layer):
    sd = fr.weight_set("stress", 1)
    ins = fr.make_inputs("floats", *SHAPE, 40)
    acts = _chain(sd, ins, mode, fault, layer)
    ref = fr.layer_reference(sd, layer, _layer_input(ins, acts, layer), mode)
    with pytest.raises(AssertionError):
        fr.check(acts[layer].value, ref, fr.TAU[mode], fault)
    # the launches before it are untouched and pass
    for before in range(layer):
        fr.check(acts[before].value, fr.layer_reference(sd, before, _layer_input(ins, acts, before), mode),
                 fr.TAU[mode], fr.LAYER_NAMES[before])
