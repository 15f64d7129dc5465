"""Float64 references for each launch of the forward pass (test helper; imported by the CPU and GPU suites).

``wn_debug_forward_layer`` (``Engine.debug_layer``) returns the output of one launch of the forward, decoded to
fp32 (``LAYER_NAMES``; 0 and 8 are the two outputs of the fused first launch).  ``layer_reference(sd, layer, a)``
evaluates that launch in float64 from the input the GPU launch consumed: the four input images for layers 0 and 8,
otherwise the decoded output of the launch before it (``INPUT_LAYER``).  Each launch is judged on its own input, so
errors do not pile up along the chain and the bar sees the launch alone.  It returns R, a magnitude M and a floor F:

* a ReLU layer: z = conv(a, W) + b, R = relu(z), M = conv(|a|, |W|) + |b|.  ReLU is 1-Lipschitz, so a bar on z holds
  unchanged for R; no ReLU has to be kept from flipping, and any weights can be used.
* the maps (layer 7): R = sigmoid(z), M = sigmoid'(z) (conv(|a|, |W|) + |b|), and F = 2^-21 R: the map is
  evaluated in fp32 (expf, one add, one division: a few ulps of R), which sigmoid'(z) M cannot cover
  where a map saturates (z = 20: sigmoid' = 2e-9 while fp32 rounds the map to 1.0).
* the gated output (``gate_reference``): R = sum_r refined_r cm_r from the GPU's own maps and refined images,
  M = sum_r |refined_r| cm_r.

The check is ``grad_reference.assert_grad_close(G, R, M + F / tau, tau)``: |G - R| <= tau M + F element by element,
with tau per mode (``TAU``).  M is the bar for every error that is relative to the products and sums of the launch:
bf16 operand splits, e4m3's relative rounding in its normal range, fp32 accumulation and the storage format.

The fp8 floor (bf16_fp8 mode only).  An e4m3 value x = e4m3(y) (cvt.rn.satfinite, |y| <= 448) has 3 mantissa bits,
normal numbers from 2^-6 and subnormals spaced 2^-9 below that:  |x - y| <= 2^-4 |y| for |y| >= 2^-6, and
|x - y| <= 2^-10 for |y| < 2^-6.  The relative part is a product error of at most 2^-13 (the corrections are 2^-9
of the main product) and is inside tau M.  The absolute part 2^-10 is not proportional to any term of M: it is what
the floor bounds.  With DESIGN section 3 and ``pack_stages_f8_kernel``, for a weight w (w_hi = bf16(w), w_lo = w - w_hi
in fp32), the layer's power-of-two scale ws (``f8_scale_finish_kernel``: max|w| of the launch in [112, 224]) and an
activation v stored as hi = bf16(v), lo8 = e4m3((v - hi) 2^9), v8 = e4m3(v), decoded as a = hi + lo8 2^-9:

* a launch that writes hi + fp8 planes stores lo8 2^-9: floor 2^-10 2^-9 = 2^-19 per output element;
* a launch that reads them computes hi w_hi + (lo8 e4m3(w ws) + v8 e4m3(w_lo ws 2^9)) 2^-9 / ws per product, so per
  product (a != 0 and w != 0; zero operands are exact):
    - e4m3(w ws):         |lo8 2^-9| 2^-10 / ws,       with |lo8 2^-9| = |a - hi| <= 2^-7 |a| + 2^-18;
    - e4m3(w_lo ws 2^9):  |v8| 2^-10 2^-9 / ws,        with |v8| <= 1.125 |a| + 2^-10;
    - e4m3(v):            2^-10 |e4m3(w_lo ws 2^9)| 2^-9 / ws  <=  2^-10 (1.125 |w_lo| + 2^-19 / ws);
  summed over the taps and input channels of each output element, as convolutions of these terms.
The bounds on |a - hi| and |v8| follow from |v - hi| <= 2^-8 |v| (bf16 rounding) and the e4m3 bound above.  bf16
has fp32's exponent range, so the bf16x3 and fp32 modes have no such floor.

``emulate_layer`` restates the kernels' operand formats in torch, every product taken exactly in float64, for the CPU
tests: the bf16 round-to-nearest split of ``split_bf16x2``; a_hi w_hi + a_lo w_hi + a_hi w_lo (the a_lo pass is zero
for inputs that are exact 8-bit levels); the fp8 form above with ws as ``f8_scale_finish_kernel`` computes it; the
first launch's v * 255 operands (snapped to a level within 2^-14) and W / 255 weights; and the output written back
in the launch's storage format.  Its faults (``FAULTS``) are the arithmetic mistakes the bar must reject.
"""
from __future__ import annotations

import types

import numpy as np
import torch
import torch.nn.functional as F

from grad_reference import assert_grad_close
from oracle import forward as ofw

# Bars of tests/test_forward_layers_gpu.py: 4x the worst (|G - R| - F) / M measured per mode on an H100 (80 GB HBM3,
# 700 W limit; DESIGN section 2): 6.4e-7 (fp32, refiners.conv2), 1.24e-5 (bf16x3, cmg.conv2 of the trained weights)
# and 9.7e-5 (bf16_fp8, refiners.conv1, whose output is stored as hi + e4m3((v - hi) 2^9)).
TAU = {"fp32": 2.6e-6, "bf16x3": 5e-5, "bf16_fp8": 3.9e-4}
MODES = tuple(TAU)

LAYER_NAMES = ["cmg.conv1", "cmg.conv2", "cmg.conv3", "cmg.conv4", "cmg.conv5", "cmg.conv6", "cmg.conv7",
               "cmg.conv8 (maps)", "refiners.conv1", "refiners.conv2", "refiners.conv3"]
CHANNELS = (128, 128, 128, 64, 64, 64, 64, 3, 96, 96, 9)
INPUT_LAYER = {0: None, 1: 0, 2: 1, 3: 2, 4: 3, 5: 4, 6: 5, 7: 6, 8: None, 9: 8, 10: 9}
MAPS, REFINED = 7, 10
# the launches with an fp8 form (kSpecs f8: C2, C3, C5, C6, C7, R2) and those that write hi + fp8 planes for them
# (writes_f8: L1, C2, C4, C5, C6), by debug-layer number
READS_F8 = {1, 2, 4, 5, 6, 9}
WRITES_F8 = {0, 8, 1, 3, 4, 5}


def _blocks(layer):
    """[(state-dict prefix, kernel, input, output channel offset)] of one launch; input is a channel slice of the
    previous output, or ("images", r) for a first layer: cat[x, wb, he, gc] (r = None) or cat[x, image r + 1]."""
    if layer < 8:
        name, _, _, k = ofw.CMG_LAYERS[layer]
        return [(f"cmg.{name}", k, ("images", None) if layer == 0 else slice(None), 0)]
    name, _, cout, k = ofw.REFINER_LAYERS[layer - 8]
    return [(f"{ref}.{name}", k, ("images", r) if layer == 8 else slice(32 * r, 32 * r + 32), cout * r)
            for r, ref in enumerate(ofw.REFINERS)]


def _block_input(src, a):
    if isinstance(src, tuple):
        r = src[1]
        return torch.cat(list(a), 1) if r is None else torch.cat([a[0], a[1 + r]], 1)
    return a[:, src]


def f8_ws(sd, layer):
    """ws of the launch, as f8_scale_finish_kernel computes it from max|w| over all its weights."""
    mx = max(float(sd[p + ".weight"].abs().max()) for p, _, _, _ in _blocks(layer))
    return float(np.exp2(np.floor(np.log2(np.float32(224.0) / np.float32(max(mx, 1e-30))))))


def _w_lo(w):
    w = w.float()
    return (w - w.bfloat16().float()).double()


def layer_reference(sd, layer, a, mode=None, device=None):
    """R, M and F (module docstring) of launch ``layer`` in float64 on ``device`` (default: the input's).  ``a`` is
    the list of four input images for layers 0 and 8, else the decoded output of INPUT_LAYER[layer].  The fp8
    floor is added for mode == "bf16_fp8"."""
    first = layer in (0, 8)
    device = device or (a[0].device if first else a.device)
    a = [t.detach().to(device, torch.float64) for t in a] if first else a.detach().to(device, torch.float64)
    f8 = mode == "bf16_fp8"
    ws = f8_ws(sd, layer) if f8 and layer in READS_F8 else None
    zs, ms, fs = [], [], []
    for prefix, k, src, _ in _blocks(layer):
        w = sd[prefix + ".weight"].to(device, torch.float64)
        b = sd[prefix + ".bias"].to(device, torch.float64)
        x = _block_input(src, a)
        zs.append(F.conv2d(x, w, b, padding=k // 2))
        ms.append(F.conv2d(x.abs(), w.abs(), b.abs(), padding=k // 2))
        fl = torch.zeros_like(zs[-1])
        if ws is not None:
            nz = (x != 0).double()
            per_a = nz * ((2.0 ** -7 * x.abs() + 2.0 ** -18) * 2.0 ** -10 / ws      # e4m3(w ws)
                          + (1.125 * x.abs() + 2.0 ** -10) * 2.0 ** -19 / ws)       # e4m3(w_lo ws 2^9)
            fl = fl + F.conv2d(per_a, (w != 0).double(), padding=k // 2)
            fl = fl + 2.0 ** -10 * F.conv2d(nz, 1.125 * _w_lo(w).abs() + 2.0 ** -19 / ws * (w != 0).double(),
                                            padding=k // 2)                          # e4m3(v)
        fs.append(fl)
    z, M, Fl = torch.cat(zs, 1), torch.cat(ms, 1), torch.cat(fs, 1)
    if f8 and layer in WRITES_F8:
        Fl = Fl + 2.0 ** -19
    if layer == MAPS:
        R = torch.sigmoid(z)
        return types.SimpleNamespace(R=R, M=R * torch.sigmoid(-z) * M, F=Fl + 2.0 ** -21 * R, z=z)
    return types.SimpleNamespace(R=F.relu(z), M=M, F=Fl, z=z)


def gate_reference(maps, refined):
    """out = sum_r refined_r cm_r (net.py:104-108) in float64 from the given maps (N,3,H,W) and refined images (N,9,H,W),
    with M = sum_r |refined_r| cm_r and no floor."""
    cm = maps.detach().double()
    rf = refined.detach().to(cm.device, torch.float64)
    R = sum(rf[:, 3 * r:3 * r + 3] * cm[:, r:r + 1] for r in range(3))
    M = sum(rf[:, 3 * r:3 * r + 3].abs() * cm[:, r:r + 1] for r in range(3))
    return types.SimpleNamespace(R=R, M=M, F=torch.zeros_like(R))


def check(G, ref, tau, name=""):
    """|G - R| <= tau M + F element by element (grad_reference.assert_grad_close names the worst element)."""
    return assert_grad_close(G.detach().to(ref.R.device, torch.float64), ref.R, ref.M + ref.F / tau, tau, name)


def excess(G, ref):
    """The measured value tau is set from: max over the elements of (|G - R| - F)+ / M."""
    err = ((G.detach().to(ref.R.device, torch.float64) - ref.R).abs() - ref.F).clamp_min(0)
    ratio = torch.where(ref.M > 0, err / ref.M.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return ratio.max().item() if ratio.numel() else 0.0


# ------------------------------------------------------------------ weight sets and inputs
def trained_state_dict():
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trained_synthetic_400ep.npz")
    with np.load(path) as z:
        return {k: torch.from_numpy(z[k]) for k, _ in ofw.state_dict_spec()}


def graded_state_dict(sd):
    """Output channel c of every ReLU layer that feeds another convolution (weights and bias) scaled by 2^-k,
    k = c mod 13, and the next layer's weights of input channel c by 2^k: the same function up to rounding (ReLU
    commutes with a positive scale), with activations down in e4m3's subnormal range and each layer's weights
    spanning more than the range of its one fp8 scale."""
    sd = {k: v.clone() for k, v in sd.items()}
    chains = [[f"cmg.{n}" for n, _, _, _ in ofw.CMG_LAYERS]] + \
             [[f"{ref}.{n}" for n, _, _, _ in ofw.REFINER_LAYERS] for ref in ofw.REFINERS]
    for chain in chains:
        for prev, nxt in zip(chain[:-1], chain[1:]):
            s = 2.0 ** -(torch.arange(sd[prev + ".bias"].numel()) % 13).float()
            sd[prev + ".weight"] *= s[:, None, None, None]
            sd[prev + ".bias"] *= s
            sd[nxt + ".weight"] *= (1 / s)[None, :, None, None]
    return sd


# ------------------------------------------------------------------ producer / consumer pairs of the e4m3 range guard
# P -> Q: the layer whose output Q reads.  FP8_PRODUCERS write hi + fp8 planes in the default mode (WRITES_F8), so
# the range guard of their epilogue decides whether Q's fp8 pass may run; cmg.conv4 is computed in cmg.conv3's
# epilogue (kFmtFuse1x1).  PLAIN_PRODUCERS write hi / lo planes (or registers): nothing of their output is converted
# to e4m3, so they must never raise the flag.
FP8_PRODUCERS = ("cmg.conv1",) + tuple(f"{r}.conv1" for r in ofw.REFINERS) + ("cmg.conv2", "cmg.conv4", "cmg.conv5",
                                                                              "cmg.conv6")
PLAIN_PRODUCERS = ("cmg.conv3", "cmg.conv7") + tuple(f"{r}.conv2" for r in ofw.REFINERS)
E4M3_MAX = 448.0


def _chain(producer):
    stack, name = producer.split(".")
    names = [n for n, _, _, _ in (ofw.CMG_LAYERS if stack == "cmg" else ofw.REFINER_LAYERS)]
    return stack, names, names.index(name)


def consumer(producer):
    """The state-dict prefix of the layer that reads ``producer``'s output."""
    stack, names, i = _chain(producer)
    return f"{stack}.{names[i + 1]}"


def producer_layer(producer):
    """(debug-layer number, output channel slice) of ``producer``'s activation in ``Engine.debug_layer``'s dump."""
    stack, _, i = _chain(producer)
    if stack == "cmg":
        return i, slice(None)
    r = ofw.REFINERS.index(stack)
    return 8 + i, slice(32 * r, 32 * r + 32)


def pushed_state_dict(sd, producer, g):
    """P's weights and bias times g, its consumer Q's weights times 1 / g: the same function, since ReLU commutes with
    a positive scale.  With g a power of two, and nothing leaving fp32's normal range, the bf16 splits, every fp32
    product and sum, the bias add, ReLU and the power-of-two fp8 weight scales (ws, s_c) commute with it as well, so
    only P's own activations change, by exactly g.  ``producer``: a state-dict prefix (``cmg.conv4``,
    ``gc_refiner.conv1``) or a tuple of them."""
    sd = {k: v.clone() for k, v in sd.items()}
    for p in (producer,) if isinstance(producer, str) else producer:
        q = consumer(p)
        sd[p + ".weight"] *= g
        sd[p + ".bias"] *= g
        sd[q + ".weight"] *= 1.0 / g
    return sd


def boundary_state_dict(sd, producer, channel, value):
    """Every weight and bias upstream of P and P's own weights zeroed, and P's bias of output ``channel`` set to
    ``value``: on any input that channel of P's activation is exactly relu(value) at every pixel."""
    sd = {k: v.clone() for k, v in sd.items()}
    stack, names, i = _chain(producer)
    for n in names[:i]:
        sd[f"{stack}.{n}.weight"].zero_()
        sd[f"{stack}.{n}.bias"].zero_()
    sd[producer + ".weight"].zero_()
    sd[producer + ".bias"][channel] = value
    return sd


# a block of fp8 planes whose largest value is below this is recomputed in bf16x3 (kF8LowMax, DESIGN 4.2)
F8_LOW_MAX = 2.0 ** -6


def trip_gains(m, threshold=E4M3_MAX):
    """(g_below, g_above) for a producer whose largest activation is m > 0: g_above the smallest power of two with
    g_above m > threshold, g_below = g_above / 2, so that g_below m lies in (threshold / 2, threshold].  At 448 they
    are g_safe and g_trip; at F8_LOW_MAX, g_above keeps P in range and g_below trips the low end."""
    k = int(np.floor(np.log2(threshold / m))) + 1
    while 2.0 ** k * m <= threshold:
        k += 1
    while 2.0 ** (k - 1) * m > threshold:
        k -= 1
    return 2.0 ** (k - 1), 2.0 ** k


def guard_margin(x, threshold=E4M3_MAX):
    """|x - threshold| / threshold: how far a pushed maximum is from one of the guard's thresholds."""
    return abs(x - threshold) / threshold


def weight_set(name, seed=0):
    return {"stress": lambda: ofw.synthetic_state_dict(seed, 3.0),
            "default": lambda: ofw.synthetic_state_dict(seed, 1.0),
            "trained": trained_state_dict,
            "graded": lambda: graded_state_dict(ofw.synthetic_state_dict(seed, 3.0))}[name]()


WEIGHT_SETS = ("stress", "default", "trained", "graded")
INPUT_KINDS = ("levels", "floats", "dark_floats", "dark_levels")


def make_inputs(kind, n, h, w, seed):
    """Four (n,3,h,w) fp32 images: 8-bit levels u / 255 (the first launch's 2-pass form), random floats (3-pass),
    floats in [0, 0.02], or levels with a near-black region (0..5) over the left three quarters."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(4):
        if kind in ("levels", "dark_levels"):
            u = torch.randint(0, 256, (n, 3, h, w), generator=g)
            if kind == "dark_levels":
                u[..., : max(1, 3 * w // 4)] %= 6
            out.append(u.float() / 255)
        else:
            t = torch.rand(n, 3, h, w, generator=g)
            out.append(t * 0.02 if kind == "dark_floats" else t)
    return out


# ------------------------------------------------------------------ emulation of the kernels' arithmetic
FAULTS = ("drop_w_lo", "drop_w_lo_second_block", "skip_lo", "f8_scale_2x", "shifted_tap", "swapped_channels",
          "zero_edge_row", "zero_edge_column", "bf16_channel", "tf32_weights")


def _f32(t):
    return t.float().double()


def _bf16(t):
    return t.float().bfloat16().double()


def _e4m3(t):
    return t.float().clamp(-448, 448).to(torch.float8_e4m3fn).double()


def _split(v):
    hi = _bf16(v)
    return hi, _bf16(v - hi)


class Act(types.SimpleNamespace):
    """An emulated activation: ``value`` (what the debug call decodes) and the operand planes a consumer reads:
    bf16 hi / lo, or hi / lo8 = e4m3((v - hi) 2^9) / v8 = e4m3(v)."""


def _store(v, fmt):
    """v (fp32 values) written as `fmt`: "f32", "bf16" (hi + lo) or "f8" (hi + fp8 planes)."""
    if fmt == "f32":
        return Act(value=v)
    hi = _bf16(v)
    if fmt == "bf16":
        lo = _bf16(v - hi)
        return Act(value=hi + lo, hi=hi, lo=lo)
    lo8 = _e4m3((v - hi) * 512)
    return Act(value=hi + lo8 / 512, hi=hi, lo8=lo8, v8=_e4m3(v))


def _first_operands(images):
    """pack_inputs_kernel: fl32(v * 255), snapped to the level within 2^-14; exact = every value is a level."""
    f = _f32(torch.cat(list(images), 1).double() * 255)
    r = torch.round(f)
    snap = ((f - r).abs() <= 2.0 ** -14) & (r >= 0) & (r <= 255)
    return torch.where(snap, r, f), bool(snap.all())


def emulate_layer(sd, layer, a, mode, fault=None):
    """The output of launch ``layer`` in ``mode`` as an Act.  ``a``: the four images (layers 0 and 8), else the Act
    of INPUT_LAYER[layer].  ``fault`` (one of FAULTS) makes the launch compute it wrongly."""
    first = layer in (0, 8)
    f8_in = mode == "bf16_fp8" and layer in READS_F8
    if first:
        ops, exact = _first_operands(a)
        ops = ops.double()
        if mode == "fp32":
            ops, exact = torch.cat([t.double() for t in a], 1), False
        planes = Act(value=ops)
        if mode != "fp32":
            planes.hi, planes.lo = _split(ops)
    else:
        planes, exact = a, False
    ws = f8_ws(sd, layer) if f8_in else None
    zs = []
    for prefix, k, src, _ in _blocks(layer):
        w = sd[prefix + ".weight"].double()
        b = sd[prefix + ".bias"].double()
        if first:
            w = _f32(w / 255) if mode != "fp32" else w
            cols = slice(None) if src[1] is None else [0, 1, 2, 3 * (src[1] + 1), 3 * (src[1] + 1) + 1,
                                                       3 * (src[1] + 1) + 2]
            pick = lambda t: t[:, cols]
        else:
            pick = lambda t: t[:, src]
        if fault == "shifted_tap":  # tap (k // 2, 0) reads one pixel to the right
            w = w.clone()
            w[..., k // 2, 1] += w[..., k // 2, 0]
            w[..., k // 2, 0] = 0
        conv = lambda x, ww: F.conv2d(x, ww, None, padding=k // 2)
        if mode == "fp32":
            if fault == "tf32_weights":
                w = (w.float().view(torch.int32) & ~0x1FFF).view(torch.float32).double()
            z = conv(pick(planes.value), w)
        else:
            w_hi = _bf16(w)
            w_lo = _f32(w - w_hi) if f8_in else _bf16(w - w_hi)
            z_main = conv(pick(planes.hi), w_hi)
            if f8_in:
                z_corr = (conv(pick(planes.lo8), _e4m3(w * ws)) + conv(pick(planes.v8), _e4m3(w_lo * ws * 512))) / (512 * ws)
                if fault == "f8_scale_2x":  # both accumulators are dequantised by the one scale
                    z_main, z_corr = 2 * z_main, 2 * z_corr
            else:
                z_corr = conv(pick(planes.hi), w_lo) if fault not in ("drop_w_lo", "drop_w_lo_second_block") else 0
                if fault == "drop_w_lo_second_block":  # one 16 x 16 tile's second m64 block: columns 8..15 of tile 0
                    full = conv(pick(planes.hi), w_lo)
                    z_corr = full.clone()
                    z_corr[..., :16, 8:16] = 0
                if not (exact or fault == "skip_lo"):
                    z_corr = z_corr + conv(pick(planes.lo), w_hi)
            z = z_main + z_corr
            if fault == "bf16_channel":  # output channel 0 from a_hi x w_hi alone
                z = z.clone()
                z[:, 0] = z_main[:, 0]
        zs.append(z + b.view(1, -1, 1, 1))
    v = _f32(torch.cat(zs, 1))
    if fault == "swapped_channels":
        v = v[:, [1, 0] + list(range(2, v.shape[1]))]
    if layer == MAPS:
        return _store(_f32(torch.sigmoid(v)), "f32")
    v = F.relu(v)
    if fault == "zero_edge_row":
        v = v.clone()
        v[..., -1, :] = 0
    if fault == "zero_edge_column":
        v = v.clone()
        v[..., :, -1] = 0
    if mode == "fp32" or layer == REFINED:
        return _store(v, "f32")
    return _store(v, "f8" if mode == "bf16_fp8" and layer in WRITES_F8 else "bf16")


def emulate_gate(maps, refined):
    """The gate epilogue in fp32: (r0 c0 + r1 c1) + r2 c2, every product and sum rounded."""
    p = [_f32(refined[:, 3 * r:3 * r + 3] * maps[:, r:r + 1]) for r in range(3)]
    return _f32(_f32(p[0] + p[1]) + p[2])
