"""Float64 references for each launch of the training backward (test helper; imported by the CPU and GPU suites).

``wn_debug_backward_layer`` (``Engine.debug_backward_layer``) returns one buffer of the backward, decoded to fp32
(``BUFFERS``): the saved forward activations, the two seeds and the output of each of the 11 data-gradient launches.
Every reference here is computed from the GPU's own decoded buffers, so each launch is judged on exactly the input it
consumed: the ReLU decisions of the forward are the GPU's (no ReLU can flip against the reference, and any weights
can be used), and no launch inherits the error of the launches before it.  Each reference returns R and a magnitude M
on the same terms, and the check is ``grad_reference.assert_grad_close(G, R, M, tau)``, |G - R| <= tau M element by
element; where M is 0 (a masked pixel, a padding channel) G must be exactly 0.0.

* Seeds (``seed_reference``): seed_kernel's gate, maps and refine formulas from grad_out and the
  GPU's cm and refined; M is the same products in absolute values.
* Data gradient of a launch (``dgrad_reference``): R = mask * conv_transpose(g, W), M = mask * conv_transpose(|g|, |W|),
  g the decoded buffer the launch read, mask = (the GPU's saved input activation > 0) (none for the two launches
  with respect to the packed input).  The refiners' conv2 launch is block-diagonal over the three refiners; their
  conv3 launch maps 9 to 96 channels and their conv1 launch adds the three refiners' x columns.
* Weight and bias gradients (``param_reference``): dW[o][c][tap] = sum over n and px of g[o] a[c][px + tap] (zero
  padding), db = sum g, M the same sums in absolute values, with g the gradient the weight-gradient GEMM consumed
  (the seed, or the next launch's masked output) and a the GPU's saved input (act0 / 255 for the first layers:
  ``extract`` scales by 1/255; refiner r's conv1 reads packed channels 0..2 and 3(r+1)..3(r+1)+2).
* The input-gradient fold (``fold_reference``): extract_input_grads_kernel adds the decoded outputs of the two
  first-layer launches of the whole network, and copies the one of a sub-module.

The bars (``TAU``, ``wgrad_tau``; DESIGN section 4.3).  A data-gradient launch is the forward kernel in bf16x3 on
decoded operands: g_hi w_hi + g_lo w_hi + g_hi w_lo with fp32 accumulation, stored as bf16 hi + lo.  A weight
gradient adds g_hi a_hi + g_lo a_hi + g_hi a_lo over all the pixels one CTA owns in one fp32 accumulator per element,
then the CTAs' partial sums in fp32.  Its error grows with the length of that sum, so its bar is a function of P, the
pixels one partial sum covers (``wgrad_pixels``).

``emulate_*`` restate the kernels' operand formats in torch, every product taken exactly in float64, for the CPU
tests; ``FAULTS`` are the mistakes the bar must reject.
"""
from __future__ import annotations

import types

import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

import forward_reference as fr
from grad_reference import PARAM_NAMES, assert_grad_close
from oracle import forward as ofw

BUFFERS = ["act0", "a1", "a2", "a3", "a4", "a5", "a6", "a7", "cm", "r1", "r2", "refined", "g8", "gr3",
           "kD8", "kD7", "kD6", "kD5", "kD4", "kD3", "kD2", "kDR3", "kDR2", "kD1", "kDR1"]
NUMBER = {b: i for i, b in enumerate(BUFFERS)}
CHANNELS = dict(zip(BUFFERS, (16, 128, 128, 128, 64, 64, 64, 64, 3, 96, 96, 9, 16, 16,
                              64, 64, 64, 64, 128, 128, 128, 96, 96, 32, 32)))
DGRAD = BUFFERS[14:]
SAVED = BUFFERS[:12]
# the stacks of wn_debug_backward_layer: -1 the whole network, 0 the confidence maps, 1 one refiner
STACKS = {"all": -1, "cmg": 0, "refiner": 1}
_CMG_ONLY = {"a1", "a2", "a3", "a4", "a5", "a6", "a7", "cm", "g8", "kD8", "kD7", "kD6", "kD5", "kD4", "kD3", "kD2", "kD1"}


def stack_buffers(stack):
    """The buffers of a stack's training pass, in BUFFERS order."""
    if stack == "all":
        return list(BUFFERS)
    return [b for b in BUFFERS if b == "act0" or (b in _CMG_ONLY) == (stack == "cmg")]


# the cmg launch of convolution c (1-based) and its input gradient / mask buffers
_CMG_DGRAD = {"kD8": 8, "kD7": 7, "kD6": 6, "kD5": 5, "kD4": 4, "kD3": 3, "kD2": 2, "kD1": 1}
DGRAD_INPUT = {"kD8": "g8", "kD7": "kD8", "kD6": "kD7", "kD5": "kD6", "kD4": "kD5", "kD3": "kD4", "kD2": "kD3",
               "kD1": "kD2", "kDR3": "gr3", "kDR2": "kDR3", "kDR1": "kDR2"}
DGRAD_MASK = {"kD8": "a7", "kD7": "a6", "kD6": "a5", "kD5": "a4", "kD4": "a3", "kD3": "a2", "kD2": "a1", "kD1": None,
              "kDR3": "r2", "kDR2": "r1", "kDR1": None}
# (ks, nci, tpg) of each launch's weight-gradient GEMM (conv_bwd.cu kDSpecs) and the convolutions it serves
WGRAD_CFG = {"kD8": (3, 64, 4), "kD7": (3, 64, 4), "kD6": (5, 64, 4), "kD5": (7, 64, 4), "kD4": (1, 128, 1),
             "kD3": (3, 128, 2), "kD2": (5, 128, 2), "kDR3": (3, 96, 2), "kDR2": (5, 96, 2), "kD1": (7, 16, 16),
             "kDR1": (7, 16, 16)}


def _cmg(c):
    name, cin, cout, k = ofw.CMG_LAYERS[c - 1]
    return f"cmg.{name}", cin, cout, k


def _first_cols(r):
    """Packed input channels refiner r's conv1 reads: cat[x, input r + 1]."""
    return [0, 1, 2, 3 * (r + 1), 3 * (r + 1) + 1, 3 * (r + 1) + 2]


def dgrad_blocks(li):
    """[(state-dict prefix, kernel, input-gradient channels, output channels)] of data-gradient launch li."""
    if li in _CMG_DGRAD:
        prefix, cin, cout, k = _cmg(_CMG_DGRAD[li])
        return [(prefix, k, slice(0, cout), list(range(cin)))]
    out = []
    for r, ref in enumerate(ofw.REFINERS):
        if li == "kDR3":
            out.append((f"{ref}.conv3", 3, slice(3 * r, 3 * r + 3), list(range(32 * r, 32 * r + 32))))
        elif li == "kDR2":
            out.append((f"{ref}.conv2", 5, slice(32 * r, 32 * r + 32), list(range(32 * r, 32 * r + 32))))
        else:
            out.append((f"{ref}.conv1", 7, slice(32 * r, 32 * r + 32), _first_cols(r)))
    return out


def wgrad_specs():
    """{state-dict prefix: (launch li whose weight-gradient GEMM computes it, g buffer, g channels, a buffer, a
    channels, scale)} for the 17 convolutions, in state-dict order."""
    spec = {}
    for li, c in sorted(_CMG_DGRAD.items(), key=lambda kv: kv[1]):
        prefix, cin, cout, _ = _cmg(c)
        g = "g8" if c == 8 else f"kD{c + 1}"
        a = "act0" if c == 1 else f"a{c - 1}"
        spec[prefix] = (li, g, slice(0, cout), a, list(range(cin)), 1 / 255 if c == 1 else 1.0)
    for r, ref in enumerate(ofw.REFINERS):
        spec[f"{ref}.conv1"] = ("kDR1", "kDR2", slice(32 * r, 32 * r + 32), "act0", _first_cols(r), 1 / 255)
        spec[f"{ref}.conv2"] = ("kDR2", "kDR3", slice(32 * r, 32 * r + 32), "r1", list(range(32 * r, 32 * r + 32)), 1.0)
        spec[f"{ref}.conv3"] = ("kDR3", "gr3", slice(3 * r, 3 * r + 3), "r2", list(range(32 * r, 32 * r + 32)), 1.0)
    assert [p + ".weight" for p in spec] == PARAM_NAMES[::2]
    return spec


WGRAD_SPECS = wgrad_specs()


def stack_params(stack, which=0):
    """The state-dict prefixes of the convolutions whose gradients a stack's backward writes, in state-dict order
    (the order of the gradient tensors the library's backward calls take)."""
    prefixes = list(WGRAD_SPECS)
    if stack == "cmg":
        return [p for p in prefixes if p.startswith("cmg.")]
    if stack == "refiner":
        return [p for p in prefixes if p.startswith(ofw.REFINERS[which] + ".")]
    return prefixes


# ------------------------------------------------------------------ the bars
# 4x the worst |G - R| / M measured on an H100 (80 GB HBM3, 700 W limit) over tests/test_backward_layers_gpu.py
# (DESIGN section 4.3).  seed: seed_kernel's gate / maps / refine (7.7e-6); dgrad: the 11 data-gradient launches
# (1.90e-5, the refiners' conv3 launch); bias: the 34 bias-gradient reductions (2.9e-7); fold:
# extract_input_grads_kernel's fp32 sums of the decoded first-layer gradients (1.19e-7, one rounding).
TAU = {"seed": 3.1e-5, "dgrad": 7.6e-5, "bias": 1.2e-6, "fold": 4.8e-7}
# The weight gradients.  Up to a few thousand pixels per partial sum the error is that of the bf16x3 products and
# the bf16 hi + lo operands (worst 1.45e-5, flat in P); WGRAD_TAU0 is 4x that.  Beyond, the fp32 accumulation shows:
# one CTA's partial sum of P pixels takes 3P/16 accumulator updates (one per K = 16 step of each of the three
# passes), and each can lose up to 2^-23 of the running sum, which is at most M (the tensor cores' accumulation is
# not documented to round to nearest, so the unit of a truncating add).  The bar adds that bound, (3P/16) 2^-23;
# the worst measured, 1.37e-4 at P = 22976 (1 x 385 x 577, the refiners' conv2), is 27% of it, 1/4.2 of the bar.
WGRAD_TAU0 = 5.8e-5


def wgrad_tau(pixels):
    """The weight-gradient bar for a GEMM whose CTAs each sum ``pixels`` pixels (``wgrad_pixels``)."""
    return WGRAD_TAU0 + 3 * pixels / 16 * 2.0 ** -23


def wgrad_geometry(li, n, h, w, sm_count):
    """(tiles per CTA, tile rows TY, pixel splits) of launch li's weight-gradient GEMM (conv_bwd.cu WgradCfg and
    launch_wgrad)."""
    ks, nci, tpg = WGRAD_CFG[li]

    def stage_bytes(ty):
        return (2 * 16 * ty * 16 * 16 + 2 * (nci // 8) * (ty + ks - 1) * (16 + ks - 1) * 16 + 1023) // 1024 * 1024

    ty = 8 if 2 * stage_bytes(8) + 2048 <= 227 * 1024 else 4
    groups = -(-ks * ks // tpg)
    tiles = -(-w // 16) * -(-h // ty) * n
    splits = max(1, min(sm_count // groups, tiles))
    if splits * groups > 192:
        splits = 192 // groups
    return -(-tiles // splits), ty, splits


def wgrad_pixels(li, n, h, w, sm_count):
    """P: the pixel positions one CTA's partial sum covers (16 x TY per tile)."""
    per_cta, ty, _ = wgrad_geometry(li, n, h, w, sm_count)
    return per_cta * 16 * ty


# ------------------------------------------------------------------ references
def _f64(t, device):
    return t.detach().to(device, torch.float64)


def seed_reference(stack, grad, cm=None, refined=None, which=0, device=None):
    """{"g8": ns(R, M), "gr3": ns(R, M)} of the stack's seed kernel, 16 channels each (the unused ones R = M = 0)."""
    device = device or grad.device
    go = _f64(grad, device)
    n, _, h, w = go.shape
    out = {}
    if stack in ("all", "cmg"):
        c = _f64(cm, device)
        R = torch.zeros(n, 16, h, w, dtype=torch.float64, device=device)
        M = torch.zeros_like(R)
        d = c * (1 - c)
        if stack == "all":
            rf = _f64(refined, device)
            for r in range(3):
                R[:, r] = (go * rf[:, 3 * r:3 * r + 3]).sum(1) * d[:, r]
                M[:, r] = (go * rf[:, 3 * r:3 * r + 3]).abs().sum(1) * d[:, r]
        else:
            R[:, :3] = go * d
            M[:, :3] = R[:, :3].abs()
        out["g8"] = types.SimpleNamespace(R=R, M=M)
    if stack in ("all", "refiner"):
        rf = _f64(refined, device)
        R = torch.zeros(n, 16, h, w, dtype=torch.float64, device=device)
        M = torch.zeros_like(R)
        for r in range(3):
            if stack == "refiner" and r != which:
                continue
            on = (rf[:, 3 * r:3 * r + 3] > 0).double()
            v = go * (_f64(cm, device)[:, r:r + 1] if stack == "all" else 1.0) * on
            R[:, 3 * r:3 * r + 3] = v
            M[:, 3 * r:3 * r + 3] = v.abs()
        out["gr3"] = types.SimpleNamespace(R=R, M=M)
    return out


def dgrad_reference(sd, li, g, mask=None, device=None):
    """R and M of data-gradient launch li from its decoded input gradient g and the saved activation that masks it."""
    device = device or g.device
    g = _f64(g, device)
    n, _, h, w = g.shape
    R = torch.zeros(n, CHANNELS[li], h, w, dtype=torch.float64, device=device)
    M = torch.zeros_like(R)
    for prefix, k, gch, cols in dgrad_blocks(li):
        wt = sd[prefix + ".weight"].to(device, torch.float64)
        R[:, cols] += F.conv_transpose2d(g[:, gch], wt, padding=k // 2)
        M[:, cols] += F.conv_transpose2d(g[:, gch].abs(), wt.abs(), padding=k // 2)
    if mask is not None:
        on = (_f64(mask, device) > 0).double()
        R, M = R * on, M * on
    return types.SimpleNamespace(R=R, M=M)


def param_reference(prefix, bufs, device=None):
    """(weight ns(R, M), bias ns(R, M)) of one convolution from the decoded buffers ``bufs`` {name: tensor}."""
    li, gname, gch, aname, acols, scale = WGRAD_SPECS[prefix]
    device = device or bufs[gname].device
    g = _f64(bufs[gname], device)[:, gch]
    a = _f64(bufs[aname], device)[:, acols] * scale
    k = WGRAD_CFG[li][0]
    shape = (g.shape[1], a.shape[1], k, k)
    wR = nn_grad.conv2d_weight(a, shape, g, padding=k // 2)
    wM = nn_grad.conv2d_weight(a.abs(), shape, g.abs(), padding=k // 2)
    return (types.SimpleNamespace(R=wR, M=wM),
            types.SimpleNamespace(R=g.sum((0, 2, 3)), M=g.abs().sum((0, 2, 3))))


def fold_reference(stack, kd1=None, kdr1=None, which=0):
    """The input gradients from the decoded first-layer launches: [ns(R, M)] for x, wb, he, gc (the whole network,
    the cmg) or x, xbar (refiner `which`)."""
    if stack == "all":
        a, b = kd1.double(), kdr1.double()
        return [types.SimpleNamespace(R=a[:, 3 * t:3 * t + 3] + b[:, 3 * t:3 * t + 3],
                                      M=a[:, 3 * t:3 * t + 3].abs() + b[:, 3 * t:3 * t + 3].abs()) for t in range(4)]
    src = (kd1 if stack == "cmg" else kdr1).double()
    slots = range(4) if stack == "cmg" else (0, which + 1)
    return [types.SimpleNamespace(R=src[:, 3 * s:3 * s + 3], M=src[:, 3 * s:3 * s + 3].abs()) for s in slots]


def check(G, ref, tau, name=""):
    return assert_grad_close(G.detach().to(ref.R.device, torch.float64), ref.R, ref.M, tau, name)


def ratio(G, ref):
    """max |G - R| / M (inf where M == 0 and G != R)."""
    err = (G.detach().to(ref.R.device, torch.float64) - ref.R).abs()
    r = torch.where(ref.M > 0, err / ref.M.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return r.max().item() if r.numel() else 0.0


# ------------------------------------------------------------------ emulation of the kernels' arithmetic
FAULTS = ("mask_right", "mask_down", "mask_pair_swap", "no_mask", "mask_tile_row", "mask_tile_column",
          "unrotated_taps", "drop_g_lo", "drop_a_lo", "missing_tile", "zero_tap_group", "bias_hi_only",
          "seed_no_one_minus_cm", "seed_no_refined_mask", "first_layer_no_255", "first_layer_255_twice",
          "refiner_next_channels")
_f32, _bf16, _store, Act = fr._f32, fr._bf16, fr._store, fr.Act


def emulate_forward(sd, ins):
    """The saved buffers of the bf16x3 training forward (forward_reference.emulate_layer) as Acts."""
    ops, exact = fr._first_operands(ins)
    ops = torch.cat([ops.double(), torch.zeros_like(ops[:, :4]).double()], 1)
    hi, lo = fr._split(ops)
    bufs = {"act0": Act(value=hi + lo, hi=hi, lo=lo)}
    acts = {}
    for layer in range(11):
        src = ins if fr.INPUT_LAYER[layer] is None else acts[fr.INPUT_LAYER[layer]]
        acts[layer] = fr.emulate_layer(sd, layer, src, "bf16x3")
    for layer in range(7):
        bufs[f"a{layer + 1}"] = acts[layer]
    bufs.update(cm=acts[7], r1=acts[8], r2=acts[9], refined=acts[10])
    return bufs


def emulate_seeds(stack, grad, bufs, which=0, fault=None):
    """seed_kernel's gate / maps / refine in fp32, stored as 16-channel bf16 hi + lo buffers."""
    go = _f32(grad.double())
    n, _, h, w = go.shape
    out = {}
    if stack in ("all", "cmg"):
        c = bufs["cm"].value
        v = torch.zeros(n, 16, h, w, dtype=torch.float64)
        one_minus = torch.ones_like(c) if fault == "seed_no_one_minus_cm" else _f32(1 - c)
        for r in range(3):
            if stack == "all":
                rf = bufs["refined"].value
                dot = _f32(go[:, 0] * rf[:, 3 * r])
                dot = _f32(dot + _f32(go[:, 1] * rf[:, 3 * r + 1]))
                dot = _f32(dot + _f32(go[:, 2] * rf[:, 3 * r + 2]))
            else:
                dot = go[:, r]
            v[:, r] = _f32(_f32(dot * c[:, r]) * one_minus[:, r])
        out["g8"] = _store(v, "bf16")
    if stack in ("all", "refiner"):
        rf = bufs["refined"].value
        v = torch.zeros(n, 16, h, w, dtype=torch.float64)
        for r in range(3):
            if stack == "refiner" and r != which:
                continue
            on = torch.ones_like(rf[:, :3]) if fault == "seed_no_refined_mask" else (rf[:, 3 * r:3 * r + 3] > 0).double()
            scale = bufs["cm"].value[:, r:r + 1] if stack == "all" else 1.0
            v[:, 3 * r:3 * r + 3] = _f32(go * scale) * on
        out["gr3"] = _store(v, "bf16")
    return out


def _shift(t, dy, dx):
    """t[..., y + dy, x + dx], zero beyond the image."""
    out = torch.zeros_like(t)
    h, w = t.shape[-2:]
    out[..., :h - dy, :w - dx] = t[..., dy:, dx:]
    return out


def emulate_dgrad(sd, li, g, mask, fault=None):
    """Data-gradient launch li on the bf16 hi + lo gradient g (an Act) and the saved activation mask (an Act or
    None): g_hi w_hi + g_lo w_hi + g_hi w_lo with pack_stages_kernel's bf16 split of the weights, the ReLU' mask,
    the result stored as bf16 hi + lo."""
    n, _, h, w = g.hi.shape
    z = torch.zeros(n, CHANNELS[li], h, w, dtype=torch.float64)
    for prefix, k, gch, cols in dgrad_blocks(li):
        wt = sd[prefix + ".weight"].double()
        if fault == "unrotated_taps":  # the forward's taps, not rotated by 180 degrees
            wt = wt.flip(-1, -2)
        w_hi = _bf16(wt)
        w_lo = _bf16(wt - w_hi)
        ct = lambda x, ww: F.conv_transpose2d(x[:, gch], ww, padding=k // 2)
        part = ct(g.hi, w_hi) + ct(g.hi, w_lo)
        if fault != "drop_g_lo":
            part = part + ct(g.lo, w_hi)
        z[:, cols] += part
    v = _f32(z)
    if mask is not None and fault != "no_mask":
        on = (mask.value > 0).double()
        if fault == "mask_right":
            on = _shift(on, 0, 1)
        elif fault == "mask_down":
            on = _shift(on, 1, 0)
        elif fault == "mask_pair_swap":  # the two halves of each bf16 pair
            idx = torch.arange(on.shape[1]).view(-1, 2).flip(1).reshape(-1)
            on = on[:, idx]
        elif fault == "mask_tile_row":  # the last row of every 16 x 16 tile
            on = on.clone()
            on[..., 15::16, :] = 0
        elif fault == "mask_tile_column":
            on = on.clone()
            on[..., :, 15::16] = 0
        v = v * on
    return _store(v, "bf16")


def emulate_params(prefix, bufs, fault=None):
    """(weight, bias) gradients of one convolution: dense = g_hi a_hi + g_lo a_hi + g_hi a_lo summed exactly, then
    fp32 and extract's fp32 scale; the bias from hi + lo."""
    li, gname, gch, aname, acols, scale = WGRAD_SPECS[prefix]
    if fault == "refiner_next_channels" and prefix.endswith(".conv1") and not prefix.startswith("cmg."):
        acols = _first_cols((ofw.REFINERS.index(prefix.split(".")[0]) + 1) % 3)
    k, _, tpg = WGRAD_CFG[li]
    g, a = bufs[gname], bufs[aname]
    g_hi, g_lo = g.hi[:, gch], g.lo[:, gch]
    a_hi, a_lo = a.hi[:, acols], a.lo[:, acols]
    if fault == "missing_tile":  # one CTA's share: the 16 x 8 pixel tile at the origin of image 0
        keep = torch.ones_like(g_hi[:, :1])
        keep[0, :, :8, :16] = 0
        g_hi, g_lo = g_hi * keep, g_lo * keep
    shape = (g_hi.shape[1], a_hi.shape[1], k, k)
    cw = lambda x, y: nn_grad.conv2d_weight(x, shape, y, padding=k // 2)
    dense = cw(a_hi, g_hi) + cw(a_hi, g_lo)
    if fault != "drop_a_lo":
        dense = dense + cw(a_lo, g_hi)
    dense = _f32(dense)
    if fault == "zero_tap_group":  # the second tap group of the launch
        dense = dense.reshape(*shape[:2], k * k).clone()
        dense[..., tpg:2 * tpg] = 0
        dense = dense.reshape(shape)
    if scale != 1.0:
        s = float(torch.tensor(1 / 255, dtype=torch.float32))
        if fault == "first_layer_no_255":
            s = 1.0
        elif fault == "first_layer_255_twice":
            s = float(torch.tensor(s * s, dtype=torch.float32))
        dense = _f32(dense * s)
    gb = g_hi if fault == "bias_hi_only" else g_hi + g_lo
    return dense, _f32(gb.sum((0, 2, 3)))


def emulate_backward(sd, stack, grad, bufs, which=0, fault=None, fault_at=None):
    """Every buffer of the stack's backward and its parameter gradients: (bufs with the seeds and launches added,
    {prefix: (dW, db)}).  ``fault`` is applied at ``fault_at``: a seed name, a launch or a state-dict prefix."""
    bufs = dict(bufs)
    bufs.update(emulate_seeds(stack, grad, bufs, which, fault if fault_at in ("g8", "gr3") else None))
    have = stack_buffers(stack)
    for li in DGRAD:
        if li not in have:
            continue
        mask = DGRAD_MASK[li]
        bufs[li] = emulate_dgrad(sd, li, bufs[DGRAD_INPUT[li]], bufs[mask] if mask else None,
                                 fault if fault_at == li else None)
    params = {p: emulate_params(p, bufs, fault if fault_at == p else None) for p in stack_params(stack, which)}
    return bufs, params
