"""The e4m3 range guard of the default mode at every producer of fp8 planes and on every forward entry point.

Every launch that writes hi + fp8 planes for an fp8 consumer checks its activations in its epilogue (``epilogue16``:
a value above 448 raises the handle's sticky flag), and the bf16x3 chain queued behind each fp8 pass runs when the
flag is up.  These tests move each producer P's activations to the guard's threshold with
``forward_reference.pushed_state_dict`` (P times a power of two g, its consumer Q times 1 / g): the float64 result
does not change, and the bf16x3 and fp32 bits do not change either (test_range_guard_cpu.py).  g is chosen from P's
largest activation M_P in the bf16x3 dump: g_trip the smallest power of two with g M_P > 448, g_safe = g_trip / 2,
each at least 1e-3 of 448 away from it.

* g_safe: the flag stays down, every launch passes the float64 bars of test_forward_layers_gpu on its own input, the
  output is within 6e-4 of float64 and the uint8 output within one level of it.
* g_trip: the flag is up after the first call and the output is the bf16x3 output of the unpushed weights, bit for
  bit, on every entry point.
* Producers that write no fp8 planes (cmg.conv3, cmg.conv7, the refiners' conv2) pushed by 2^12 never raise it.
* One channel at exactly 448 leaves the flag down, the next float up raises it, at positions 0, 7, 8 and 15 of a
  16-channel group and in the refiners' columns of the first launch.
* A multi-pass or ragged call that trips in a later pass: the passes before keep their fp8 bits, the tripping pass
  and every later one return bf16x3 bits (DESIGN 4.2).
"""
import types

import numpy as np
import pytest
import torch

import forward_reference as fr
from oracle import forward as ofw
from oracle import preprocess as opre
from test_forward_layers_gpu import _check_case
from test_gpu_parity import _assert_close, _assert_u8_close, _inputs_from_rgb

pytestmark = pytest.mark.gpu

SHAPES = [(2, 40, 56), (3, 37, 53)]   # partial 8 x 24 and 16 x 24 tiles
WEIGHTS = ["stress", "trained", "default"]   # trained: cmg.conv5 is zero on these images
MARGIN = 1e-3
TILE = (24, 32)                       # several windows per image on the windowed entry points
NEXT_448 = float(np.nextafter(np.float32(448), np.float32(np.inf)))


def _model(precision):
    from waternet_b200.net import WaterNet
    return WaterNet(precision=precision).cuda().eval()


@pytest.fixture(scope="module")
def models():
    return {p: _model(p) for p in ("bf16_fp8", "bf16x3", "fp32")}


def _load(m, sd):
    """New weights: packed at the next call, which also clears the range flag."""
    m.load_state_dict(sd, strict=True)
    return m


def _overflowed(m):
    torch.cuda.synchronize()
    return m.engine().f8_overflowed()


def _run(m, cu):
    with torch.no_grad():
        return m(*cu)


def _reference64(sd, cu):
    """WaterNet.forward in float64 on the GPU (oracle.forward's layers)."""
    sdc = {k: v.cuda().double() for k, v in sd.items()}
    x, wb, he, gc = (t.double() for t in cu)
    with torch.no_grad():
        cm = ofw.confidence_maps(sdc, x, wb, he, gc)
        return sum(ofw.refine(sdc, r, x, xbar) * cm[:, i:i + 1]
                   for i, (r, xbar) in enumerate(zip(ofw.REFINERS, (wb, he, gc))))


def _max_activation(m16, cu, producer, per_image=False):
    """P's largest activation in the bf16x3 dump of launch producer_layer(P) (m16: a bf16x3 model)."""
    layer, cols = fr.producer_layer(producer)
    from waternet_b200 import _lib
    a = m16.engine().debug_layer(*cu, layer=layer, mode=_lib.MODE_BF16X3)[:, cols]
    return a.amax(dim=(1, 2, 3)).tolist() if per_image else a.max().item()


def _safe_margins(m):
    """How far g M_P is from 448 at g_safe and g_trip, and from F8_LOW_MAX at the two gains around it (none for a
    producer whose activations are all zero)."""
    if m <= 0:
        return [1.0]
    return [fr.guard_margin(g * m) for g in fr.trip_gains(m)] + \
        [fr.guard_margin(g * m, fr.F8_LOW_MAX) for g in fr.trip_gains(m, fr.F8_LOW_MAX)]


def _live(b, producer):
    """P's M_P, or a skip where P's activations are all zero on these inputs: no gain brings them to 448."""
    if b.maxima[producer] <= 0:
        pytest.skip(f"{producer} is zero everywhere on these inputs with these weights")
    return b.maxima[producer]


_BASES = {}


def _base(models, weights, shape):
    """Weights, images (the first seed whose pushed maxima all keep MARGIN from 448), their float64, bf16x3, fp32
    and default-mode outputs and each fp8 producer's M_P."""
    key = (weights, shape)
    if key in _BASES:
        return _BASES[key]
    sd = fr.weight_set(weights, 2)
    n, h, w = shape
    m16 = _load(models["bf16x3"], sd)
    for seed in range(100, 160, 6):
        rgbs = np.stack([ofw.synthetic_image(seed + i, h, w, "smooth" if i % 2 else "noise") for i in range(n)])
        ins = _inputs_from_rgb(list(rgbs))
        cu = [t.cuda() for t in ins]
        maxima = {p: _max_activation(m16, cu, p) for p in fr.FP8_PRODUCERS}
        if min(min(_safe_margins(v)) for v in maxima.values()) >= MARGIN:
            break
    else:
        pytest.fail(f"no input seed keeps every pushed maximum {MARGIN} from 448")
    b = types.SimpleNamespace(sd=sd, ins=ins, cu=cu, frames=torch.from_numpy(rgbs).cuda(), maxima=maxima,
                              ref=_reference64(sd, cu), plain=_run(m16, cu))
    b.fp32 = _run(_load(models["fp32"], sd), cu)
    b.fp8 = _run(_load(models["bf16_fp8"], sd), cu)
    assert not _overflowed(models["bf16_fp8"])
    assert not torch.equal(b.fp8, b.plain), "the default mode computes the bf16x3 bits: nothing to tell apart"
    _BASES[key] = b
    return b


# ------------------------------------------------------------------ each fp8 producer at g_safe and g_trip
@pytest.mark.parametrize("producer", fr.FP8_PRODUCERS)
@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("weights", WEIGHTS)
def test_fp8_producer_at_the_edge_of_the_e4m3_range(models, weights, shape, producer):
    b = _base(models, weights, shape)
    m_p = _live(b, producer)
    g_safe, g_trip = fr.trip_gains(m_p)
    assert min(_safe_margins(m_p)) >= MARGIN
    m = models["bf16_fp8"]
    # g_safe: in range, the default mode's own bits within its bars
    sd = fr.pushed_state_dict(b.sd, producer, g_safe)
    worst = {}
    _check_case(_load(m, sd), sd, "bf16_fp8", b.ins, worst, f"{weights} {shape} {producer} g_safe={g_safe}")
    out = _run(m, b.cu)
    assert not _overflowed(m)
    rel = _assert_close(out.cpu().numpy(), b.ref.cpu().numpy(), 6e-4)
    u8 = m.engine().enhance(b.frames, mode=m._mode())
    assert not _overflowed(m)
    _assert_u8_close(u8.cpu().numpy(), opre.ten2arr(b.ref.cpu().numpy()), share=0.10)
    layer = fr.producer_layer(producer)[0]
    print(f"{weights} {shape} {producer}: M_P={m_p:.4g} g_safe=2^{int(np.log2(g_safe))} g_trip=2^{int(np.log2(g_trip))}"
          f" worst launch at g_safe {max(v for k, v in worst.items() if k != 'gate'):.2e}"
          f" ({producer} {worst[layer]:.2e}), output {rel:.2e}")
    # g_trip: the call that trips returns the bf16x3 bits of the original weights, and so does the uint8 path
    sd = fr.pushed_state_dict(b.sd, producer, g_trip)
    out = _run(_load(m, sd), b.cu)
    assert _overflowed(m)
    assert torch.equal(out, b.plain)
    u8 = _load(m, sd).engine().enhance(b.frames, mode=m._mode())
    assert _overflowed(m)
    assert np.array_equal(u8.cpu().numpy(), opre.ten2arr(b.plain.cpu().numpy()))


@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("weights", WEIGHTS)
def test_bf16x3_and_fp32_bits_do_not_move(models, weights, shape):
    """g_trip and 2^-12 on every pair: the bf16x3 and fp32 outputs are those of the original weights, bit for bit."""
    b = _base(models, weights, shape)
    for producer in fr.FP8_PRODUCERS:
        for g in (fr.trip_gains(b.maxima[producer])[1] if b.maxima[producer] > 0 else 2.0 ** 12, 2.0 ** -12):
            sd = fr.pushed_state_dict(b.sd, producer, g)
            for precision, want in (("bf16x3", b.plain), ("fp32", b.fp32)):
                m = _load(models[precision], sd)
                assert torch.equal(_run(m, b.cu), want), (producer, g, precision)
                assert not _overflowed(m)


@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("weights", WEIGHTS)
def test_producers_without_fp8_planes_never_raise_the_flag(models, weights, shape):
    """cmg.conv3 (fused with cmg.conv4 in the forward, its own launch in the debug dump), cmg.conv7 and the
    refiners' conv2 (one launch, one fp8 weight scale: pushed together) times 2^12: the flag stays down, every launch
    passes its bars and the default-mode output is that of the original weights bit for bit."""
    b = _base(models, weights, shape)
    m = models["bf16_fp8"]
    for producer in ("cmg.conv3", "cmg.conv7", tuple(f"{r}.conv2" for r in ofw.REFINERS)):
        sd = fr.pushed_state_dict(b.sd, producer, 2.0 ** 12)
        _check_case(_load(m, sd), sd, "bf16_fp8", b.ins, {}, f"{weights} {shape} {producer}")
        assert torch.equal(_run(m, b.cu), b.fp8), producer
        assert not _overflowed(m)


# ------------------------------------------------------------------ one channel at the threshold
BOUNDARY = [(p, c) for p, n in (("cmg.conv1", 128), ("cmg.conv2", 128), ("cmg.conv4", 64), ("cmg.conv5", 64),
                                ("cmg.conv6", 64)) for c in (0, 16 + 7, n // 2 + 8, n - 1)] + \
           [("wb_refiner.conv1", 8), ("gc_refiner.conv1", 15)]


@pytest.mark.parametrize("producer,channel", BOUNDARY)
def test_one_channel_at_the_threshold(models, producer, channel):
    """Zero levels in, every weight up to P's zeroed: P's channel holds exactly its bias.  448 leaves the flag down
    (P's dump holds 448 in that channel), nextafter(448) and +inf raise it (the bf16x3 bits, NaNs equal).  A NaN bias is made 0
    by the ReLU (fmaxf) in every mode before any e4m3 conversion: flag down, the bits of a zero bias."""
    cu = [torch.zeros(1, 3, 40, 56, device="cuda") for _ in range(4)]
    sd0 = fr.weight_set("stress", 2)
    m, m16 = models["bf16_fp8"], models["bf16x3"]
    sd = fr.boundary_state_dict(sd0, producer, channel, 448.0)
    out = _run(_load(m, sd), cu)
    assert not _overflowed(m) and torch.isfinite(out).all()
    layer, cols = fr.producer_layer(producer)
    assert (m.engine().debug_layer(*cu, layer=layer, mode=m._mode())[:, cols][:, channel] == 448).all()
    for value in (NEXT_448, float("inf")):
        sd = fr.boundary_state_dict(sd0, producer, channel, value)
        out = _run(_load(m, sd), cu)
        assert _overflowed(m), value
        torch.testing.assert_close(out, _run(_load(m16, sd), cu), rtol=0, atol=0, equal_nan=True)
    out = _run(_load(m, fr.boundary_state_dict(sd0, producer, channel, float("nan"))), cu)
    assert not _overflowed(m)
    assert torch.equal(out, _run(_load(m, fr.boundary_state_dict(sd0, producer, channel, 0.0)), cu))


# ------------------------------------------------------------------ entry points
def _trip_sd(models, producer):
    """Stress weights with ``producer`` pushed to trip on both the level images and float inputs of its base."""
    b = _base(models, "stress", SHAPES[0])
    floats = [t.cuda() for t in fr.make_inputs("floats", *SHAPES[0], 61)]
    m16 = _load(models["bf16x3"], b.sd)
    m_floats = _max_activation(m16, floats, producer)
    g = max(fr.trip_gains(b.maxima[producer])[1], fr.trip_gains(m_floats)[1])
    for m_p in (b.maxima[producer], m_floats):   # both kinds of input leave the range by the margin
        assert g * m_p >= 448 * (1 + MARGIN), (producer, g, m_p)
    return b, floats, fr.pushed_state_dict(b.sd, producer, g)


@pytest.mark.parametrize("producer", ["cmg.conv4", "gc_refiner.conv1"])
def test_every_entry_point_returns_the_bf16x3_bits_when_it_trips(models, producer):
    from waternet_b200.net import ConfidenceMapGenerator, Refiner
    b, floats, sd = _trip_sd(models, producer)
    m, m16 = models["bf16_fp8"], _load(models["bf16x3"], sd)
    e16 = m16.engine()
    mode, mode16 = m._mode(), m16._mode()

    def trips(call):
        """call(engine, mode) on fresh weights in the default mode, the flag up after it, its result bit for bit
        that of the bf16x3 model."""
        got = call(_load(m, sd).engine(), mode)
        assert _overflowed(m), call.__name__
        want = call(e16, mode16)
        torch.cuda.synchronize()
        for a, w in zip(got if isinstance(got, list) else [got], want if isinstance(want, list) else [want]):
            assert torch.equal(a, w), call.__name__

    def forward_levels(e, md):
        return e.forward(*b.cu, md)

    def forward_floats(e, md):
        return e.forward(*floats, md)

    def enhance(e, md):
        f32 = torch.empty(b.frames.shape[0], 3, *b.frames.shape[1:3], device="cuda")
        return [e.enhance(b.frames, mode=md, out_f32=f32).clone(), f32]

    def enhance_tiled(e, md):
        return e.enhance_tiled(b.frames, tile=TILE, mode=md).clone()

    def enhance_ragged(e, md):
        imgs = [b.frames[1, 3:, 5:].contiguous()] + list(b.frames)
        return [t.clone() for t in e.enhance_ragged(imgs, tile=TILE, mode=md)]

    def forward_tiled(e, md):
        return e.forward_tiled(*floats, tile=TILE, mode=md)

    def forward_ragged(e, md):
        items = [tuple(floats), tuple(t[1:, :, 2:, 4:] for t in b.cu)]
        return e.forward_ragged(items, TILE, md)

    for call in (forward_levels, forward_floats, enhance, enhance_tiled, enhance_ragged, forward_tiled,
                 forward_ragged):
        trips(call)
    # WaterNet.forward and forward_many through the module
    for ins in (b.cu, floats):
        got = _run(_load(m, sd), ins)
        assert _overflowed(m) and torch.equal(got, _run(m16, ins))
    items = [tuple(floats), tuple(t[1:, :, 1:, 3:] for t in b.cu)]
    with torch.no_grad():
        got = _load(m, sd).forward_many(*zip(*items))
        assert _overflowed(m)
        want = m16.forward_many(*zip(*items))
    assert all(torch.equal(a, w) for a, w in zip(got, want))
    # the sub-module on its own, default precision, whole and in windows (a fresh module: its own engine and flag)
    stack = producer.split(".")[0]
    cls, args = (ConfidenceMapGenerator, b.cu) if stack == "cmg" else (Refiner, (b.cu[0], b.cu[3]))
    own = {k[len(stack) + 1:]: v for k, v in sd.items() if k.startswith(stack + ".")}
    for tile in (None, TILE):
        outs = {}
        for precision in ("default", "bf16x3"):
            sub = cls()
            sub.load_state_dict(own)
            sub.precision, sub.tile = precision, tile
            sub = sub.cuda().eval()
            with torch.no_grad():
                r = sub(*args)
            outs[precision] = torch.cat(r, 1) if isinstance(r, tuple) else r
            torch.cuda.synchronize()
            assert sub._engine_and_slot(args[0])[0].f8_overflowed() == (precision == "default"), (tile, precision)
        assert torch.equal(outs["default"], outs["bf16x3"]), tile


def test_cuda_graph_captured_in_range_replays_the_bf16x3_chain(models):
    """An Enhancer graph captured on a dark batch (gc_refiner.conv1 in range, flag down) and replayed on a bright
    batch that trips it: the replay returns the bf16x3 bytes and raises the flag."""
    from waternet_b200.api import Enhancer
    producer = "gc_refiner.conv1"
    b, _, sd = _trip_sd(models, producer)
    rng = np.random.default_rng(5)
    dark = rng.integers(0, 4, b.frames.shape, dtype=np.uint8)
    bright = b.frames.cpu().numpy()
    m, m16 = models["bf16_fp8"], _load(models["bf16x3"], sd)
    _load(m, sd)
    enh = Enhancer(m, depth=1)
    first = enh(dark)                              # warm-up and capture
    assert not _overflowed(m) and enh._slots[0].graph is not None
    graph = enh._slots[0].graph
    assert np.array_equal(enh(dark), first)        # replay, in range
    got = enh(bright)                              # replay of the same graph on the tripping batch
    assert enh._slots[0].graph is graph
    assert _overflowed(m)
    assert np.array_equal(got, Enhancer(m16, cuda_graph=False)(bright))


# ------------------------------------------------------------------ multi-pass and ragged calls that trip in a later pass
def test_multi_pass_and_ragged_calls_that_trip_in_a_later_pass(models):
    """[dark, bright, dark], one image per pass, g between the images' maxima (gc_refiner.conv1): image 0 keeps its
    fp8 bits, images 1 and 2 return their bf16x3 bits (the flag is sticky and every later pass's bf16x3 chain runs).
    A batch that stays in range keeps the fp8 bits of every image."""
    producer = "gc_refiner.conv1"
    n, h, w = 3, 40, 56
    dark = fr.make_inputs("dark_floats", n, h, w, 71)
    bright = fr.make_inputs("floats", n, h, w, 72)
    cu = [torch.cat([d[:1], bb[1:2], d[2:]]).cuda() for d, bb in zip(dark, bright)]
    sd0 = fr.weight_set("stress", 2)
    m, m16 = models["bf16_fp8"], _load(models["bf16x3"], sd0)
    mx = _max_activation(m16, cu, producer, per_image=True)
    assert mx[1] >= 2 * (1 + MARGIN) * max(mx[0], mx[2]), mx
    g = fr.trip_gains(mx[1])[1]
    assert g * mx[1] >= 448 * (1 + MARGIN) and g * max(mx[0], mx[2]) <= 448 * (1 - MARGIN)
    sd = fr.pushed_state_dict(sd0, producer, g)
    _load(m, sd)
    alone = [_run(m, [t[i:i + 1] for t in cu]) for i in (0, 2)]   # the dark images in range: fp8 bits
    assert not _overflowed(m)
    m16 = _load(models["bf16x3"], sd)
    plain = _run(m16, cu)
    assert not torch.equal(alone[0], plain[:1]) and not torch.equal(alone[1], plain[2:])
    eng = m.engine()
    eng.set_chunk_pixels(h * w)
    try:
        assert eng.chunk_images(n, h, w) == 1
        dark_batch = [torch.cat([t[:1], t[2:], t[:1]]) for t in cu]
        out = _run(m, dark_batch)
        assert not _overflowed(m)
        assert torch.equal(out, torch.cat([alone[0], alone[1], alone[0]]))
        out = _run(m, cu)
        assert _overflowed(m)
    finally:
        eng.set_chunk_pixels(0)
    assert torch.equal(out[:1], alone[0]), "the pass before the one that tripped keeps its fp8 bits"
    assert torch.equal(out[1:], plain[1:]), "the tripping pass and every later pass return bf16x3 bits"
    # the ragged call: one window per image, one image per pass, in image order
    from waternet_b200.engine import ragged_plan
    items = [tuple(t[i:i + 1] for t in cu) for i in range(n)]
    assert [p["windows"][0]["img"] for p in ragged_plan([(h, w)] * n, 998, 998, h * w)] == [0, 1, 2]
    out = _load(m, sd).engine().forward_ragged(items, (998, 998), m._mode(), max_pass_pixels=h * w)
    assert _overflowed(m)
    assert torch.equal(out[0], alone[0]) and torch.equal(torch.cat(out[1:]), plain[1:])


def test_new_weights_clear_the_flag(models):
    """cmg.conv5 tripped, then the original weights: the next call runs the fp8 corrections again."""
    b = _base(models, "stress", SHAPES[0])
    m = models["bf16_fp8"]
    _run(_load(m, fr.pushed_state_dict(b.sd, "cmg.conv5", fr.trip_gains(b.maxima["cmg.conv5"])[1])), b.cu)
    assert _overflowed(m)
    out = _run(_load(m, b.sd), b.cu)
    assert not _overflowed(m)
    assert torch.equal(out, b.fp8)


# ------------------------------------------------------------------ the low end: a whole producer in e4m3's subnormals
@pytest.mark.parametrize("producer", fr.FP8_PRODUCERS)
def test_producer_in_the_subnormal_range_runs_in_bf16x3(models, producer):
    """g = 2^-12: every correction operand of P is an e4m3 subnormal or zero, which costs the default mode 1.3e-3 to
    5.3e-3 of its output.  The fp8 launches still pass their per-launch bars (whose floor covers exactly that), and
    P's consumer sees that P's block stayed below F8_LOW_MAX: the call raises the flag and returns the bf16x3 bits of
    the original weights, on tensors and on the uint8 path."""
    b = _base(models, "stress", SHAPES[0])
    sd = fr.pushed_state_dict(b.sd, producer, 2.0 ** -12)
    m = models["bf16_fp8"]
    _check_case(_load(m, sd), sd, "bf16_fp8", b.ins, {}, f"{producer} g=2^-12", forward=False)
    out = _run(_load(m, sd), b.cu)
    assert _overflowed(m)
    assert torch.equal(out, b.plain)
    u8 = _load(m, sd).engine().enhance(b.frames, mode=m._mode())
    assert _overflowed(m)
    assert np.array_equal(u8.cpu().numpy(), opre.ten2arr(b.plain.cpu().numpy()))


@pytest.mark.parametrize("producer", fr.FP8_PRODUCERS)
@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_producer_at_the_low_threshold(models, shape, producer):
    """P's largest activation just above F8_LOW_MAX = 2^-6: the flag stays down and the output is within the 1e-3
    parity bar of float64 (reported: the band's error).  Just below it: the flag is up and the output is the bf16x3
    output of the original weights bit for bit.  The record is per block, so a refiner alone trips its call."""
    b = _base(models, "stress", shape)
    m_p = b.maxima[producer]
    g_low, g_ok = fr.trip_gains(m_p, fr.F8_LOW_MAX)
    m = models["bf16_fp8"]
    out = _run(_load(m, fr.pushed_state_dict(b.sd, producer, g_ok)), b.cu)
    assert not _overflowed(m)
    rel = _assert_close(out.cpu().numpy(), b.ref.cpu().numpy(), 1e-3)
    print(f"{shape} {producer}: largest activation {g_ok * m_p:.4f}, output {rel:.2e} of float64")
    out = _run(_load(m, fr.pushed_state_dict(b.sd, producer, g_low)), b.cu)
    assert _overflowed(m)
    assert torch.equal(out, b.plain)
