"""Float64 references for the backward pass of WaterNet (test helper; imported by the CPU and GPU suites).

``reference(sd, ins, grad)`` evaluates the network of ``oracle/forward.py`` in float64 on the inputs' device and
back-propagates ``grad`` = d(loss)/d(out) through it.  Besides the gradients R of the 34 parameters and the four
input images it returns every ReLU's pre-activation z and a magnitude reference M of the same shapes as R.

M is the sum of the absolute values of the terms of the reduction that produces each gradient element, taken at
the reference values: for a convolution with input a and output gradient g (the ReLU' mask applied),
M(dW[o][c][tap]) = sum_px |g[px][o]| |a[px + tap][c]|, M(db[o]) = sum_px |g[px][o]|, and an input image's M is
sum_layers |W|^T |g| over the first-layer convolutions that read it.  For conv8 g is replaced by the magnitude
of the gate's own sum, (sum_c |grad_c| refined_c) sigmoid'(z8).  It is float64 autograd through one level of
absolute values: every convolution with |W| and |b| fed its reference input |a|, weighted by |g|.
A reduction whose products and partial sums carry a relative error u (bf16x3 products, fp32 sums) is off by a
small multiple of u times M; the gradient errors it inherits from the layers behind it enter the same sums and
stay a small multiple of u of M in practice.  (The chain bound -- the whole network with |W|, seeded with
|grad| -- is rigorous but exceeds |R| by up to 1e11 on cmg.conv1: a bar on it could not tell a zeroed gradient
from a right one.)  This holds as long as no ReLU decides differently from the reference, which the networks of
the GPU tests exclude by construction (``assert_relus_cannot_flip``).  ``assert_grad_close`` checks
|G - R| <= tau * M element by element, so an error confined to one tap, one channel, one edge row or one image
stands out even where the whole tensor's norm would hide it, and elements whose M is 0 (dead channels) must be
exactly 0.
"""
from __future__ import annotations

import types

import torch
import torch.nn.functional as F

from oracle import forward as ofw

# The bar of the GPU tests (tests/test_backward_gpu.py): 4x the worst |G - R| / M measured on an H100 (80 GB HBM3,
# 400 W limit), 3.7e-4 on cmg.conv5.weight at 1 x 385 x 577 -- a weight-gradient CTA there adds ~22k pixels' products
# into one fp32 accumulator, whose rounding error grows with the length of the sum.
TAU = 1.5e-3
# On 1 x 1 images only the centre taps see data, and the data gradients -- sums over the channels alone -- cancel
# more than usual: the errors they carry into a parameter gradient are a larger share of its M (measured: 8.7e-3 on
# cmg.conv2 for three images, 3.2e-3 on cmg.conv4 for 70000).  Their parameter gradients get 4x the larger one.
TAU_ONE_PIXEL = 3.5e-2

PARAM_NAMES = [k for k, _ in ofw.state_dict_spec()]
INPUT_NAMES = ["x", "wb", "he", "gc"]
# the 16 ReLUs of the network: cmg.conv1..conv7, then every refiner's conv1..conv3
RELU_LAYERS = [f"cmg.{name}" for name, _, _, _ in ofw.CMG_LAYERS[:-1]] + \
              [f"{ref}.{name}" for ref in ofw.REFINERS for name, _, _, _ in ofw.REFINER_LAYERS]
KERNEL = {f"cmg.{name}": k for name, _, _, k in ofw.CMG_LAYERS} | \
         {f"{ref}.{name}": k for ref in ofw.REFINERS for name, _, _, k in ofw.REFINER_LAYERS}


def _first_layer_input(layer, ins):
    """The images a first-layer convolution reads: cat[x, wb, he, gc] (cmg) or cat[x, image r+1] (refiner r)."""
    x, wb, he, gc = ins
    if layer == "cmg.conv1":
        return torch.cat([x, wb, he, gc], 1)
    if layer.endswith(".conv1"):
        return torch.cat([x, ins[1 + ofw.REFINERS.index(layer.split(".")[0])]], 1)
    return None


def _leaves(tensors, device, absolute=False):
    out = []
    for t in tensors:
        t = t.detach().to(device, torch.float64)
        out.append((t.abs() if absolute else t.clone()).requires_grad_(True))
    return out


def reference(sd, ins, grad=None, target=None, device="cpu", magnitude=True):
    """Float64 gradients of the network state dict ``sd`` at the four input images ``ins``.

    The backward is seeded with ``grad`` (d(loss)/d(out)), or is that of mse_loss(out, target).  Returns a namespace:
    out, seed (d(loss)/d(out)), grads {param: R}, input_grads [R x4], z {relu layer: pre-activation} and, with
    ``magnitude``, M {param: M}
    and M_inputs [M x4] (see the module docstring).  Everything lives on ``device``."""
    params = dict(zip(PARAM_NAMES, _leaves([sd[k] for k in PARAM_NAMES], device)))
    leaves = _leaves(ins, device)
    seen = {}   # layer -> (its input, its pre-activation)

    def conv(layer, t):
        zz = F.conv2d(t, params[layer + ".weight"], params[layer + ".bias"], padding=KERNEL[layer] // 2)
        if magnitude:
            zz.retain_grad()
        seen[layer] = (t, zz)
        return zz

    x, wb, he, gc = leaves
    t = _first_layer_input("cmg.conv1", leaves)
    for name, _, _, _ in ofw.CMG_LAYERS[:-1]:
        t = F.relu(conv(f"cmg.{name}", t))
    cm = torch.sigmoid(conv("cmg.conv8", t))
    refined = []
    for ref in ofw.REFINERS:
        t = _first_layer_input(f"{ref}.conv1", leaves)
        for name, _, _, _ in ofw.REFINER_LAYERS:
            t = F.relu(conv(f"{ref}.{name}", t))
        refined.append(t)
    out = sum(r * cm[:, i:i + 1] for i, r in enumerate(refined))
    if grad is None:
        F.mse_loss(out, target.to(device, torch.float64)).backward()
        seed = 2 * (out.detach() - target.to(device, torch.float64)) / out.numel()
    else:
        seed = grad.detach().to(device, torch.float64)
        out.backward(seed)
    res = types.SimpleNamespace(
        out=out.detach(), seed=seed, grads={k: v.grad for k, v in params.items()}, input_grads=[t.grad for t in leaves],
        z={k: zz.detach() for k, (_, zz) in seen.items() if k in RELU_LAYERS})
    if not magnitude:
        return res
    # the gate's sum over the three colour channels, in absolute values: d out / d z8_r
    cm = cm.detach()
    g8 = torch.cat([(seed.abs() * r.detach()).sum(1, keepdim=True) for r in refined], 1) * cm * (1 - cm)
    del params, leaves, out, refined, t
    pabs = dict(zip(PARAM_NAMES, _leaves([sd[k] for k in PARAM_NAMES], device, absolute=True)))
    labs = _leaves(ins, device, absolute=True)
    total = 0
    for layer, (a, zz) in seen.items():
        first = _first_layer_input(layer, labs)
        a = first if first is not None else a.detach().abs()
        g = g8 if layer == "cmg.conv8" else zz.grad.abs()
        z_abs = F.conv2d(a, pabs[layer + ".weight"], pabs[layer + ".bias"], padding=KERNEL[layer] // 2)
        total = total + (z_abs * g).sum()
    seen.clear()
    total.backward()
    res.M = {k: v.grad for k, v in pabs.items()}
    res.M_inputs = [t.grad for t in labs]
    return res


# ------------------------------------------------------------------ networks whose ReLUs cannot flip
def smooth_state_dict(seed):
    """Small weights (gain 0.2) and bias 2 on every ReLU layer: every ReLU is active everywhere."""
    sd = ofw.synthetic_state_dict(seed, 0.2)
    for key in RELU_LAYERS:
        sd[key + ".bias"] = torch.full_like(sd[key + ".bias"], 2.0)
    return sd


def dead_channels(layer):
    """Output channels that the channel-gated network switches off in ReLU layer ``layer``: every third one, the
    phase advancing from layer to layer (refiner layers ordered conv1 of all three refiners, then conv2, conv3), so
    that the pattern differs between neighbouring layers and between the refiners -- one refined channel of
    each refiner is dead, a different one in each."""
    cmg = [f"cmg.{name}" for name, _, _, _ in ofw.CMG_LAYERS[:-1]]
    order = cmg + [f"{ref}.{name}" for name, _, _, _ in ofw.REFINER_LAYERS for ref in ofw.REFINERS]
    phase = order.index(layer)
    cout = dict(ofw.state_dict_spec())[layer + ".bias"][0]
    return [c for c in range(cout) if (c + phase) % 3 == 1]


def gated_state_dict(seed):
    """The smooth network with bias -2 on the channels of ``dead_channels``: those are off everywhere, the rest
    on everywhere."""
    sd = smooth_state_dict(seed)
    for layer in RELU_LAYERS:
        sd[layer + ".bias"][dead_channels(layer)] = -2.0
    return sd


def assert_relus_cannot_flip(z, ratio=0.1):
    """The premise of a tight gradient bar: on every ReLU, min |z| >= ratio * max |z|, so the forward error of any
    evaluation (~1e-5 relative) cannot move a pre-activation across zero."""
    for name, t in z.items():
        a = t.abs()
        lo, hi = a.min().item(), a.max().item()
        assert lo >= ratio * hi, (f"{name}: min |z| = {lo:.3g} < {ratio} * max |z| = {ratio * hi:.3g}: a ReLU of this "
                                  "network could flip, the test's premise does not hold")


# ------------------------------------------------------------------ the element-wise check
def _describe(name, shape, flat):
    idx = []
    for s in reversed(shape):
        idx.append(flat % s)
        flat //= s
    idx = idx[::-1]
    if name.endswith(".weight"):
        kw = shape[3]
        return f"out channel {idx[0]}, in channel {idx[1]}, tap {idx[2] * kw + idx[3]} (ky={idx[2]}, kx={idx[3]})"
    if name.endswith(".bias"):
        return f"out channel {idx[0]}"
    return f"image {idx[0]}, channel {idx[1]}, y={idx[2]}, x={idx[3]}"


def grad_error(G, R, M):
    """max |G - R| / M over the elements (inf where M == 0 and G != R; 0 for an exact match)."""
    G = G.detach().to(R.device, torch.float64)
    err = (G - R).abs()
    ratio = torch.where(M > 0, err / M.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0))
    return ratio


def assert_grad_close(G, R, M, tau, name=""):
    """|G - R| <= tau * M element by element.  On failure the message names the worst element by (out channel,
    in channel, tap) for a weight, out channel for a bias, (image, channel, y, x) for an image gradient.
    Returns the worst |G - R| / M."""
    assert tuple(G.shape) == tuple(R.shape) == tuple(M.shape), (name, tuple(G.shape), tuple(R.shape))
    ratio = grad_error(G, R, M)
    worst = ratio.max().item() if ratio.numel() else 0.0
    if not worst <= tau:
        flat = int(ratio.argmax().item())
        bad = int((ratio > tau).sum().item())
        g = G.detach().reshape(-1)[flat].item()
        r, m = R.reshape(-1)[flat].item(), M.reshape(-1)[flat].item()
        raise AssertionError(f"{name}: {bad} of {ratio.numel()} elements off by more than tau = {tau:.1e} of M; "
                             f"worst at {_describe(name, tuple(R.shape), flat)}: got {g:.9g}, want {r:.9g}, "
                             f"|d| / M = {worst:.3e} (M = {m:.3e})")
    return worst
