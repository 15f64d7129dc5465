"""Float64 replay of the single-pass bf16 training arithmetic (WN_MODE_BF16, wn_set_train_mode).

In that mode every tensor-core product is ONE bf16 wgmma, a_hi x w_hi, accumulated in fp32, and every plane buffer
(the packed input, the activations, the seeds, the data gradients) is stored as bf16(v) with lo = 0.  The replay
takes the operands a launch read (the GPU's own decoded buffers, which are then exactly bf16), rounds the weights to
bf16 with round to nearest even as pack_stages_kernel does, and forms the exact products and sums in float64.  What
is left between the replay R and the GPU's G is the fp32 accumulation of the tensor cores (the "replay bar", in the
style of backward_reference.wgrad_tau: one possible unit of 2^-23 of M per accumulator update) and, for a stored
plane buffer, the final rounding of v to bf16 (F = 2^-8 |R|, the unit roundoff of an 8-bit significand).  The
"exact-arithmetic bar" compares with the unrounded fp32 weights instead: 2^-8 M more, the worst case of rounding the
weight of every product to bf16 (the other operand, a decoded buffer, is bf16 already); with the storage floor that
makes the two bf16 roundings of a stored value.

emulate_* restate the kernels' arithmetic with exact products (the CPU test checks that it passes the bars, and that
each of FAULTS fails the bar of the launch it targets).
"""
import types

import torch
import torch.nn.functional as F
from torch.nn import grad as nn_grad

import backward_reference as br
import forward_reference as fr
from grad_reference import assert_grad_close

_bf16, _f32 = fr._bf16, fr._f32

# the products of one accumulator update: a wgmma has K = 16
K_STEP = 16
EXACT = 2.0 ** -8
ROUND = 2.0 ** -8
# seeds: a handful of fp32 operations before the bf16 store; bias and fold: fp32 sums (backward_reference.TAU)
SEED_TAU = 2.0 ** -20


def acc_tau(k):
    """The replay bar of a launch whose output element sums k products (input channels x taps): one unit of 2^-23 of
    M per accumulator update (k / 16 of them), two more for the bias add and the epilogue."""
    return (-(-k // K_STEP) + 2) * 2.0 ** -23


def wgrad_tau(pixels):
    """The replay bar of a weight-gradient GEMM whose CTAs each sum ``pixels`` pixels (backward_reference.wgrad_pixels):
    one pass of P / 16 accumulator updates, plus 2^-21 for the fp32 sum over the CTAs and the 1/255 of a first layer."""
    return 2.0 ** -21 + pixels / K_STEP * 2.0 ** -23


# products per output element as the kernels sum them (padded input channels of the element's diagonal block x taps):
# the forward launches by forward_reference number (kSpecs cinpad / nblk), the data-gradient launches (kDSpecs kpad)
_FWD_K = {0: 16 * 49, 1: 128 * 25, 2: 128 * 9, 3: 128 * 1, 4: 64 * 49, 5: 64 * 25, 6: 64 * 9, 7: 64 * 9, 8: 16 * 49,
          9: 32 * 25, 10: 96 * 9}
_DGRAD_K = {"kD8": 16 * 9, "kD7": 64 * 9, "kD6": 64 * 25, "kD5": 64 * 49, "kD4": 64, "kD3": 128 * 9,
            "kD2": 128 * 25, "kDR3": 16 * 9, "kDR2": 32 * 25, "kD1": 128 * 49, "kDR1": 96 * 49}


def launch_tau(launch):
    """The replay bar of forward launch ``launch`` (int) or data-gradient launch ``launch`` (name)."""
    return acc_tau(_FWD_K[launch] if isinstance(launch, int) else _DGRAD_K[launch])


# ------------------------------------------------------------------ references
def _w(sd, prefix, first, rounded):
    w = sd[prefix + ".weight"].double()
    if first:  # scatter_weights_kernel folds the /255 of the first layers in fp32
        w = _f32(w / 255)
    return _bf16(w) if rounded else _f32(w)


def layer_replay(sd, layer, src, rounded=True):
    """R, M, F of forward launch ``layer`` (forward_reference numbering) from its decoded input: act0 (16 channels)
    for the first layers 0 and 8, else the decoded output of forward_reference.INPUT_LAYER[layer]."""
    a = _bf16(src.double()) if rounded else src.double()
    first = layer in (0, 8)
    zs, ms = [], []
    for r, (prefix, k, blk, _) in enumerate(fr._blocks(layer)):
        w = _w(sd, prefix, first, rounded)
        b = sd[prefix + ".bias"].double()
        if first:
            x = a[:, :12] if layer == 0 else a[:, br._first_cols(r)]
        else:
            x = a[:, blk]
        zs.append(F.conv2d(x, w, b, padding=k // 2))
        ms.append(F.conv2d(x.abs(), w.abs(), b.abs(), padding=k // 2))
    z, M = torch.cat(zs, 1), torch.cat(ms, 1)
    if layer == fr.MAPS:  # fp32 sigmoid, stored fp32
        R = torch.sigmoid(z)
        return types.SimpleNamespace(R=R, M=R * torch.sigmoid(-z) * M, F=2.0 ** -21 * R)
    R = F.relu(z)
    return types.SimpleNamespace(R=R, M=M, F=(0 if layer == fr.REFINED else ROUND) * R)


def dgrad_replay(sd, li, g, mask=None, rounded=True):
    """R, M, F of data-gradient launch li from its decoded input gradient g and the saved activation that masks it."""
    g = _bf16(g.double()) if rounded else g.double()
    n, _, h, w = g.shape
    R = torch.zeros(n, br.CHANNELS[li], h, w, dtype=torch.float64, device=g.device)
    M = torch.zeros_like(R)
    for prefix, k, gch, cols in br.dgrad_blocks(li):
        wt = sd[prefix + ".weight"].to(g.device, torch.float64)
        wt = _bf16(wt) if rounded else _f32(wt)
        R[:, cols] += F.conv_transpose2d(g[:, gch], wt, padding=k // 2)
        M[:, cols] += F.conv_transpose2d(g[:, gch].abs(), wt.abs(), padding=k // 2)
    if mask is not None:
        on = (mask.double() > 0).double()
        R, M = R * on, M * on
    return types.SimpleNamespace(R=R, M=M, F=ROUND * R.abs())


def seed_replay(stack, grad, cm, refined, which=0):
    """backward_reference.seed_reference with the bf16 store's floor."""
    out = br.seed_reference(stack, grad, cm, refined, which)
    for ref in out.values():
        ref.F = ROUND * ref.R.abs()
    return out


def exact_bar(tau):
    """The exact-arithmetic bar of a launch whose replay bar is tau."""
    return tau + EXACT


def check(G, ref, tau, name="", planes=False):
    """|G - R| <= tau M + F element by element; planes: G is a decoded plane buffer, which must be exactly bf16
    (lo = 0)."""
    G = G.detach().double().to(ref.R.device)
    if planes:
        bad = (G != _bf16(G)).sum().item()
        assert bad == 0, f"{name}: {bad} elements are not bf16 (a lo plane is not 0)"
    Fl = ref.F if torch.is_tensor(getattr(ref, "F", None)) else torch.zeros_like(ref.R)
    return assert_grad_close(G, ref.R, ref.M + Fl / tau, tau, name)


def excess(G, ref):
    """max over the elements of (|G - R| - F)+ / M: what the bar's tau is compared with."""
    G = G.detach().double().to(ref.R.device)
    Fl = ref.F if torch.is_tensor(getattr(ref, "F", None)) else torch.zeros_like(ref.R)
    err = ((G - ref.R).abs() - Fl).clamp_min(0)
    r = torch.where(ref.M > 0, err / ref.M.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return r.max().item() if r.numel() else 0.0


# ------------------------------------------------------------------ emulation of the kernels' arithmetic
FAULTS = ("a_lo_pass", "w_lo_pass", "lo_not_zeroed", "g_lo_wgrad")


def _hi(v):
    """v stored in single-pass bf16: bf16(v), lo = 0."""
    h = _bf16(v)
    return fr.Act(value=h, hi=h, lo=torch.zeros_like(h))


def _hilo(v):
    return fr._store(v, "bf16")


def emulate_forward(sd, ins, fault=None, fault_at=None):
    """The saved buffers of the single-pass training forward.  fault_at: a forward_reference layer number."""
    ops, _ = fr._first_operands(ins)
    ops = torch.cat([ops.double(), torch.zeros_like(ops[:, :4]).double()], 1)
    bufs = {"act0": _hi(ops)}
    acts = {}
    names = {7: "cm", 8: "r1", 9: "r2", 10: "refined"}
    for layer in range(11):
        first = layer in (0, 8)
        src = bufs["act0"] if first else acts[fr.INPUT_LAYER[layer]]
        f = fault if fault_at == layer else None
        if f == "a_lo_pass" and not first:  # the consumer's a_lo pass: its input kept a lo plane, and it is read
            src = _hilo(src.value_full)
        zs = []
        for r, (prefix, k, blk, _) in enumerate(fr._blocks(layer)):
            w_f = _w(sd, prefix, first, False)
            w_hi = _bf16(w_f)
            cols = (slice(0, 12) if layer == 0 else br._first_cols(r)) if first else blk
            conv = lambda x, ww: F.conv2d(x[:, cols], ww, None, padding=k // 2)
            z = conv(src.hi, w_hi)
            if f == "a_lo_pass":
                z = z + conv(src.lo, w_hi)
            if f == "w_lo_pass":
                z = z + conv(src.hi, _bf16(w_f - w_hi))
            zs.append(_f32(z) + sd[prefix + ".bias"].double().view(1, -1, 1, 1))
        v = _f32(torch.cat(zs, 1))
        if layer == fr.MAPS:
            acts[layer] = fr.Act(value=_f32(torch.sigmoid(v)))
        elif layer == fr.REFINED:
            acts[layer] = fr.Act(value=F.relu(v))
        else:
            v = F.relu(v)
            acts[layer] = _hilo(v) if f == "lo_not_zeroed" else _hi(v)
            acts[layer].value_full = v
    for layer in range(7):
        bufs[f"a{layer + 1}"] = acts[layer]
    bufs.update({names[l]: acts[l] for l in names})
    return bufs


def emulate_backward(sd, stack, grad, bufs, which=0, fault=None, fault_at=None):
    """Every buffer of the stack's single-pass backward and its parameter gradients: (bufs, {prefix: (dW, db)}).
    fault_at: a seed name, a data-gradient launch or a state-dict prefix."""
    bufs = dict(bufs)
    for name, s in br.emulate_seeds(stack, grad, bufs, which).items():  # hi + lo of the same fp32 seed
        v = s.hi + s.lo
        bufs[name] = _hilo(v) if fault == "lo_not_zeroed" and fault_at == name else _hi(v)
        bufs[name].value_full = v
    have = br.stack_buffers(stack)
    for li in br.DGRAD:
        if li not in have:
            continue
        g = bufs[br.DGRAD_INPUT[li]]
        mask = br.DGRAD_MASK[li]
        f = fault if fault_at == li else None
        z = torch.zeros(g.hi.shape[0], br.CHANNELS[li], *g.hi.shape[2:], dtype=torch.float64)
        for prefix, k, gch, cols in br.dgrad_blocks(li):
            wt = _f32(sd[prefix + ".weight"].double())
            w_hi = _bf16(wt)
            ct = lambda x, ww: F.conv_transpose2d(x[:, gch], ww, padding=k // 2)
            part = ct(g.hi, w_hi)
            if f == "w_lo_pass":
                part = part + ct(g.hi, _bf16(wt - w_hi))
            if f == "a_lo_pass":
                part = part + ct(_hilo(g.value_full).lo, w_hi)
            z[:, cols] += part
        v = _f32(z)
        if mask is not None:
            v = v * (bufs[mask].value > 0).double()
        bufs[li] = _hilo(v) if f == "lo_not_zeroed" else _hi(v)
        bufs[li].value_full = v
    params = {}
    for prefix in br.stack_params(stack, which):
        li, gname, gch, aname, acols, scale = br.WGRAD_SPECS[prefix]
        k = br.WGRAD_CFG[li][0]
        g, a = bufs[gname], bufs[aname]
        g_hi, a_hi = g.hi[:, gch], a.hi[:, acols]
        shape = (g_hi.shape[1], a_hi.shape[1], k, k)
        cw = lambda x, y: nn_grad.conv2d_weight(x, shape, y, padding=k // 2)
        dense = cw(a_hi, g_hi)
        if fault == "g_lo_wgrad" and fault_at == prefix:  # g_lo x a_hi of a gradient that kept its lo plane
            dense = dense + cw(a_hi, _hilo(g.value_full).lo[:, gch])
        dense = _f32(dense)
        if scale != 1.0:
            dense = _f32(dense * float(torch.tensor(1 / 255, dtype=torch.float32)))
        params[prefix] = (dense, _f32(g_hi.sum((0, 2, 3))))
    return bufs, params
