"""The fp8-correction layers' one-accumulator order (UmmaCfg kFmtIn8, DESIGN section 4.2), emulated in float64.

A tile of such a layer runs two phases into ONE fp32 accumulator: the correction phase adds, per (16-channel chunk,
tap), the e4m3 wgmma [e4m3(lo 2^9) | e4m3(v)] x [e4m3(w ws) ; e4m3(w_lo ws 2^9)]; the main phase then adds every
a_hi x w_hi ws 2^9 (bf16).  Hopper's fp8 wgmma adds into its accumulator with fewer bits than fp32.  NVIDIA does not
document how many, so the accumulator model here keeps ``bits`` significant bits of the running value after each e4m3
wgmma (truncation toward zero) and rounds to fp32 after each bf16 wgmma.  The argument: during the correction phase
|acc| is about 2^-8 of the launch's magnitude M, so each truncation loses about 2^-(bits + 8) M; C2's 200 updates at
bits = 13 add up to ~1e-4 M, under the bf16_fp8 bar tau = 3.9e-4.  These tests check that on every weight set, for
every launch with an fp8 form, at 13 and at 12 retained bits, and that the same model of the other order -- per
chunk, the bf16 wgmmas then the e4m3 ones into the accumulator that already holds the main product -- fails the bar.

The weight image is restated as a list of units in the order pack_stages_f8_kernel writes them (every (chunk, tap)
e4m3 unit, then every (chunk, tap) bf16 unit; within a phase, chunk pairs, and a stage is TPS taps of both chunks of
a pair), and the emulation reads it the way the producers stream it: stage it of the tile is units
[2 TPS it, 2 TPS (it + 1)), and the consumers take stage it as step it / (kk / TPS): chunk pair it / (kk / TPS) of
the correction phase, then of the main phase.
"""
import pytest
import torch
import torch.nn.functional as F

import forward_reference as fr

SHAPE = (1, 19, 24)
# launches with an fp8 form (debug-layer number -> kSpecs ks, cinpad, npad per block, nblk, tps of conv_umma.cu)
F8_SPECS = {1: (5, 128, 128, 1, 5), 2: (3, 128, 128, 1, 3), 4: (7, 64, 64, 1, 7), 5: (5, 64, 64, 1, 5),
            6: (3, 64, 64, 1, 9), 9: (5, 96, 32, 3, 5)}


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(8, n))
    yield
    torch.set_num_threads(n)


def image_units(nchunk, kk, tps):
    """pack_stages_f8_kernel's unit order: (kind, chunk, tap) of unit i of a column group's image, from the kernel's
    offset formula ((chunk / 2) (kk / tps) + tap / tps) 2 tps + (chunk % 2) tps + tap % tps within a phase."""
    units = [None] * (2 * nchunk * kk)
    for phase, kind in enumerate(("e4m3", "bf16")):
        for c in range(nchunk):
            for t in range(kk):
                u = ((c // 2) * (kk // tps) + t // tps) * 2 * tps + (c % 2) * tps + t % tps
                assert units[phase * nchunk * kk + u] is None
                units[phase * nchunk * kk + u] = (kind, c, t)
    return units


def streamed_units(nchunk, kk, tps):
    """(unit index, kind, chunk, tap) in the order the consumers issue them: the B producer sends stage it from
    it * B_STAGE (2 TPS units of npad * 32 B), the consumers read it as step it / (kk / TPS) -- chunks 2p, 2p + 1 of
    the correction phase for steps p < nchunk / 2, then of the main phase -- and issue tap by tap, both chunks."""
    out = []
    for it in range(nchunk * kk // tps):
        step, tg = divmod(it, kk // tps)
        kind, p = ("e4m3", step) if step < nchunk // 2 else ("bf16", step - nchunk // 2)
        for t in range(tps):
            for j in range(2):
                out.append((it * 2 * tps + j * tps + t, kind, 2 * p + j, tg * tps + t))
    return out


@pytest.mark.parametrize("layer", sorted(F8_SPECS))
def test_stream_order_matches_the_image(layer):
    ks, cinpad, npad, nblk, tps = F8_SPECS[layer]
    nchunk, kk = cinpad // 16, ks * ks
    units = image_units(nchunk, kk, tps)
    # stage_bytes_total: 64 B per output channel per (chunk, tap), the size of the bf16x3 image
    assert len(units) * npad * 32 == nchunk * kk * npad * 64
    streamed = streamed_units(nchunk, kk, tps)
    assert sorted(u for u, _, _, _ in streamed) == list(range(len(units)))
    # the correction phase first; a pair of chunks never straddles two diagonal blocks
    assert [k for _, k, _, _ in streamed] == ["e4m3"] * (len(units) // 2) + ["bf16"] * (len(units) // 2)
    assert (nchunk // nblk) % 2 == 0
    assert [units[u] for u, *_ in streamed] == [(k, c, t) for _, k, c, t in streamed]


def _trunc(x, bits):
    m, e = torch.frexp(x)
    return torch.ldexp(torch.trunc(m * 2.0 ** bits) / 2.0 ** bits, e)


def _per_unit(x, w, k):
    """[n, o, chunk, tap, pixels]: the products of each (16-channel chunk, tap) unit, exact in float64."""
    n, ci, h, wd = x.shape
    nchunk = -(-ci // 16)
    xp = F.pad(x, (0, 0, 0, 0, 0, nchunk * 16 - ci))
    wp = F.pad(w, (0, 0, 0, 0, 0, nchunk * 16 - ci))
    cols = F.unfold(xp, k, padding=k // 2).view(n, nchunk, 16, k * k, h * wd)
    return torch.einsum("ncjtl,ocjt->noctl", cols, wp.reshape(w.shape[0], nchunk, 16, k * k))


def emulate_two_phase(sd, layer, a, bits, interleaved=False):
    """Launch ``layer`` of the bf16_fp8 mode from the hi + fp8 planes ``a`` (a forward_reference Act): the units of the
    restated image in stream order into one accumulator per output element, then max(acc 2^-9 / ws + b, 0) in fp32
    and the launch's storage format.  interleaved: per chunk, its bf16 units, then its e4m3 units."""
    ks, cinpad, _, _, tps = F8_SPECS[layer]
    nchunk, kk = cinpad // 16, ks * ks
    ws = fr.f8_ws(sd, layer)
    n, _, h, wd = a.value.shape
    zs = []
    for blk, (prefix, k, src, _) in enumerate(fr._blocks(layer)):
        w = sd[prefix + ".weight"].double()
        b = sd[prefix + ".bias"].double()
        w_hi = fr._bf16(w)
        w_lo = fr._f32(w - w_hi)
        corr = _per_unit(a.lo8[:, src], fr._e4m3(w * ws), k) + _per_unit(a.v8[:, src], fr._e4m3(w_lo * ws * 512), k)
        main = _per_unit(a.hi[:, src], fr._bf16(w_hi * ws * 512), k)
        bnc = corr.shape[2]  # this block's chunks (a block-diagonal launch: chunk c feeds block c / (nchunk / nblk))
        acc = torch.zeros(n, w.shape[0], h * wd, dtype=torch.float64)
        order = [(kind, c % bnc, t) for _, kind, c, t in streamed_units(nchunk, kk, tps) if c // bnc == blk]
        if interleaved:
            order = [(kind, c, t) for c in range(bnc) for kind in ("bf16", "e4m3") for t in range(kk)]
        for kind, c, t in order:
            if kind == "e4m3":
                acc = _trunc(acc + corr[:, :, c, t], bits)
            else:
                acc = fr._f32(acc + main[:, :, c, t])
        v = fr._f32(fr._f32(acc * (2.0 ** -9 / ws)) + b.view(1, -1, 1))
        zs.append(v.view(n, -1, h, wd))
    v = torch.relu(torch.cat(zs, 1))
    return fr._store(v, "f8" if layer in fr.WRITES_F8 else "bf16")


def _inputs(sd, kind, seed):
    """The bf16_fp8 chain of forward_reference's emulation: the input Act of every launch."""
    ins = fr.make_inputs(kind, *SHAPE, seed)
    acts = {}
    for layer in range(11):
        src = ins if fr.INPUT_LAYER[layer] is None else acts[fr.INPUT_LAYER[layer]]
        acts[layer] = fr.emulate_layer(sd, layer, src, "bf16_fp8")
    return acts


@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
def test_two_phase_order_passes_the_bar(weights):
    """Every launch with an fp8 form, with 13 and with 12 bits kept by the e4m3 wgmma's adds."""
    sd = fr.weight_set(weights, 1)
    for i, kind in enumerate(("floats", "levels")):
        acts = _inputs(sd, kind, 50 + i)
        for layer in F8_SPECS:
            a = acts[fr.INPUT_LAYER[layer]]
            ref = fr.layer_reference(sd, layer, a.value, "bf16_fp8")
            for bits in (13, 12):
                got = emulate_two_phase(sd, layer, a, bits)
                fr.check(got.value, ref, fr.TAU["bf16_fp8"], f"{weights} {kind} bits={bits} {fr.LAYER_NAMES[layer]}")


@pytest.mark.parametrize("layer", [1, 4, 9])
def test_interleaved_order_fails_the_bar(layer):
    sd = fr.weight_set("stress", 1)
    a = _inputs(sd, "floats", 60)[fr.INPUT_LAYER[layer]]
    ref = fr.layer_reference(sd, layer, a.value, "bf16_fp8")
    fr.check(emulate_two_phase(sd, layer, a, 13).value, ref, fr.TAU["bf16_fp8"], "two-phase")
    with pytest.raises(AssertionError):
        fr.check(emulate_two_phase(sd, layer, a, 13, interleaved=True).value, ref, fr.TAU["bf16_fp8"], "interleaved")
