"""The exact references of the e4m3 range-guard tests (test_range_guard_gpu.py), checked without a GPU.

``forward_reference.pushed_state_dict`` multiplies a producer P's weights and bias by a power of two g and its
consumer Q's weights by 1 / g.  The network computes the same function, and in the bf16x3 and fp32 arithmetic of the
kernels (``forward_reference.emulate_layer``: every operand split and rounding restated) the same bits, with P's own
activations scaled by exactly g.  In the default mode only the e4m3 operands break that, and only where they are
subnormal or saturated: that is a property of the format, which the operand planes show element by element.
``boundary_state_dict`` puts exactly a chosen value in one channel of P, and ``trip_gains`` picks the powers of two
that keep P's largest activation just inside e4m3's range or push it just outside.
"""
import numpy as np
import pytest
import torch

import forward_reference as fr
from oracle import forward as ofw

SHAPE = (1, 12, 19)
PRODUCERS = fr.FP8_PRODUCERS + fr.PLAIN_PRODUCERS
GAINS = [2.0 ** k for k in (-12, -7, -1, 1, 6, 12)]


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(8, n))
    yield
    torch.set_num_threads(n)


def _chain(sd, ins, mode):
    acts = {}
    for layer in range(11):
        src = ins if fr.INPUT_LAYER[layer] is None else acts[fr.INPUT_LAYER[layer]]
        acts[layer] = fr.emulate_layer(sd, layer, src, mode)
    return acts


def _output(acts):
    return fr.emulate_gate(acts[fr.MAPS].value, acts[fr.REFINED].value)


def test_producer_tables():
    """Every launch that writes fp8 planes has its producers listed, every other ReLU layer that feeds a convolution
    is a negative control, and each pair is the producer's next layer."""
    layers = {fr.producer_layer(p)[0] for p in fr.FP8_PRODUCERS}
    assert layers == fr.WRITES_F8
    assert not {fr.producer_layer(p)[0] for p in fr.PLAIN_PRODUCERS} & fr.WRITES_F8
    assert fr.consumer("cmg.conv4") == "cmg.conv5" and fr.consumer("ce_refiner.conv1") == "ce_refiner.conv2"
    assert fr.producer_layer("gc_refiner.conv1") == (8, slice(64, 96))
    assert fr.producer_layer("ce_refiner.conv2") == (9, slice(32, 64))


@pytest.mark.parametrize("producer", PRODUCERS)
def test_pushed_weights_compute_the_same_function(producer):
    """The float64 oracle of the pushed weights equals that of the original weights to 1e-12 relative, g = 2^-12 to
    2^12."""
    sd = fr.weight_set("stress", 4)
    ins = fr.make_inputs("floats", *SHAPE, 7)
    ref = ofw.waternet_forward(sd, *ins, dtype=torch.float64)
    for g in GAINS:
        out = ofw.waternet_forward(fr.pushed_state_dict(sd, producer, g), *ins, dtype=torch.float64)
        assert (out - ref).abs().max() <= 1e-12 * ref.abs().max(), (producer, g)


@pytest.mark.parametrize("mode", ["bf16x3", "fp32"])
@pytest.mark.parametrize("producer", PRODUCERS)
def test_pushed_weights_give_the_same_bits(producer, mode):
    """In the emulated bf16x3 and fp32 arithmetic P's activation is g times the original one exactly, and Q's output,
    every later launch and the gated output are bit for bit those of the original weights."""
    sd = fr.weight_set("stress", 4)
    ins = fr.make_inputs("levels", *SHAPE, 8)
    base = _chain(sd, ins, mode)
    layer, cols = fr.producer_layer(producer)
    for g in (2.0 ** -12, 2.0 ** 12):
        acts = _chain(fr.pushed_state_dict(sd, producer, g), ins, mode)
        assert torch.equal(acts[layer].value[:, cols], g * base[layer].value[:, cols]), (producer, g)
        for later in range(11):
            if later != layer:
                assert torch.equal(acts[later].value, base[later].value), (producer, g, fr.LAYER_NAMES[later])
        assert torch.equal(_output(acts), _output(base))


def _exact_e4m3(x):
    """e4m3 values strictly inside the normal range, 2^-6 < |x| < 448: whatever x rounded to them was normal and not
    saturated (2^-6 itself can be a subnormal rounded up)."""
    return (x.abs() > 2.0 ** -6) & (x.abs() < fr.E4M3_MAX)


@pytest.mark.parametrize("producer", fr.FP8_PRODUCERS)
def test_fp8_planes_scale_exactly_outside_subnormals_and_saturation(producer):
    """The default mode's planes of the pushed P: hi is g times the original everywhere; lo8 = e4m3((v - hi) 2^9) and
    v8 = e4m3(v) are g times the original wherever the original and g times it are both normal and below 448, and
    differ where they are not (g = 2^-12 drives them into the subnormals, 2^8 past 448).  Q's e4m3 weights are the same bytes."""
    sd = fr.weight_set("stress", 4)
    ins = fr.make_inputs("levels", *SHAPE, 9)
    base = _chain(sd, ins, "bf16_fp8")
    layer, cols = fr.producer_layer(producer)
    q_layer = {0: 1, 8: 9, 1: 2, 3: 4, 4: 5, 5: 6}[layer]
    for g in (2.0 ** -12, 2.0 ** -3, 2.0 ** 8):
        sdg = fr.pushed_state_dict(sd, producer, g)
        act = fr.emulate_layer(sdg, layer, ins if layer in (0, 8) else base[fr.INPUT_LAYER[layer]], "bf16_fp8")
        b = base[layer]
        assert torch.equal(act.hi[:, cols], g * b.hi[:, cols])
        for plane in ("lo8", "v8"):
            mine, orig = getattr(act, plane)[:, cols], getattr(b, plane)[:, cols]
            exact = (_exact_e4m3(orig) & _exact_e4m3(g * orig)) | ((orig == 0) & (mine == 0))
            assert exact.any(), (producer, g, plane)
            assert torch.equal(mine[exact], g * orig[exact]), (producer, g, plane)
        v8, v8_orig = act.v8[:, cols], b.v8[:, cols]
        if g < 1:
            assert not torch.equal(v8, g * v8_orig), "no subnormal operand: the check would see nothing"
        if g > 1:
            assert (v8.abs() == fr.E4M3_MAX).any() and not torch.equal(v8, g * v8_orig)
        if q_layer in fr.READS_F8 and fr.consumer(producer).split(".")[0] == "cmg":
            # Q's weights times 1 / g, its power-of-two scale ws times g: e4m3(w ws) is unchanged
            assert fr.f8_ws(sdg, q_layer) == g * fr.f8_ws(sd, q_layer)


@pytest.mark.parametrize("producer", fr.FP8_PRODUCERS + fr.PLAIN_PRODUCERS)
def test_boundary_state_dict_puts_the_value_in_one_channel(producer):
    """P's chosen channel is exactly the value at every pixel in float64, the others relu of their bias."""
    sd = fr.weight_set("stress", 4)
    ins = [t.double() for t in fr.make_inputs("floats", *SHAPE, 10)]
    layer, cols = fr.producer_layer(producer)
    for channel, value in ((0, 448.0), (15, float(np.nextafter(np.float32(448), np.float32(np.inf)))), (7, 3.5)):
        sdb = fr.boundary_state_dict(sd, producer, channel, value)
        a = _reference_chain(sdb, ins, layer)[:, cols]
        assert (a[:, channel] == value).all(), (producer, channel, value)
        others = [c for c in range(a.shape[1]) if c != channel]
        want = torch.relu(sdb[producer + ".bias"].double())[others].view(1, -1, 1, 1)
        assert torch.equal(a[:, others], want.expand_as(a[:, others]))
    # a NaN bias: float64 carries it (torch's ReLU propagates NaN); the kernels' ReLU (fmaxf) makes it 0
    a = _reference_chain(fr.boundary_state_dict(sd, producer, 8, float("nan")), ins, layer)[:, cols]
    assert a[:, 8].isnan().all()


def _reference_chain(sd, ins, upto):
    """The float64 activation of debug layer ``upto``: layer_reference chained from the input images."""
    path = [upto]
    while fr.INPUT_LAYER[path[-1]] is not None:
        path.append(fr.INPUT_LAYER[path[-1]])
    a = ins
    for layer in reversed(path):
        a = fr.layer_reference(sd, layer, a).R
    return a


def test_trip_gains_on_synthetic_maxima():
    """g_safe m in (224, 448], g_trip = 2 g_safe, powers of two, at exact powers of two and around them."""
    rng = np.random.default_rng(0)
    ms = [1.0, 448.0, 7.0, 7.0 * (1 + 2.0 ** -20), 7.0 * (1 - 2.0 ** -20), 1e-3, 3e5, 224.0, 448.0 * (1 + 1e-7)]
    ms += list(np.exp(rng.uniform(np.log(1e-4), np.log(1e6), 200)))
    for m in ms:
        safe, trip = fr.trip_gains(m)
        assert trip == 2 * safe and np.log2(safe) == np.round(np.log2(safe)), m
        assert 224.0 < safe * m <= 448.0 and trip * m > 448.0, m
    assert fr.trip_gains(7.0) == (64.0, 128.0)           # 64 x 7 = 448 is inside: the guard trips above 448
    assert fr.trip_gains(448.0) == (1.0, 2.0)
    assert fr.trip_gains(7.0 * (1 + 2.0 ** -20)) == (32.0, 64.0)
    assert fr.guard_margin(448.0) == 0 and abs(fr.guard_margin(447.552) - 1e-3) < 1e-12
    # the low end: g_below M in (2^-7, 2^-6] trips, g_above M in (2^-6, 2^-5] stays in range
    for m in ms:
        below, above = fr.trip_gains(m, fr.F8_LOW_MAX)
        assert above == 2 * below and 2.0 ** -7 < below * m <= 2.0 ** -6 < above * m, m
    assert fr.trip_gains(1.0, fr.F8_LOW_MAX) == (2.0 ** -6, 2.0 ** -5)
