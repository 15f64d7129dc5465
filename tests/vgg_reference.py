"""Float64 references of the VGG19 perceptual loss (test helper; imported by the CPU and GPU suites): the VGG
counterpart of forward_reference.py / backward_reference.py.

Weight sets (``weights(name)``, 16 (weight, bias) pairs in ``features`` order, fp32 on the CPU):
  zero_bias  the PerceptualModel(pretrained=False) weights: torchvision's init, every bias 0;
  biased     seeded He-scaled weights whose biases are drawn at BIAS_SPREAD of each layer's pre-activation spread on a
             noise image, so that some channels are off and some on almost everywhere, as with trained weights.

Image kinds (``pair(kind, n, h, w, seed)``): "noise" (out uniform, ref a perturbed copy), "flat" (out with flat
patches, some at exactly 0 and 1, so that the pools meet tied positive maxima) and ``probe_pair`` (ref == out except
for a few 3 x 3 patches).

``chain`` is the float64 backward of the loss from the GPU's whole-image seed, through the GPU's saved ReLU' masks
and the pool routes of its saved outputs: the reference of every windowed d(out), because each window's share passes
through activations that are bit for bit the whole-image ones (DESIGN.md 4.12, window rule).  ``absolute=True``
gives the per-element magnitude M of d(out) that its bar scales with.
"""
import functools

import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
# (conv index or -1 for a pool, level, channels) of the 20 forward launches, and (cin, cout) of the 16 convolutions:
# waternet_b200.engine.VGG_STEPS / VGG_CONVS, restated so that this module imports without the library
STEPS = ((0, 0, 64), (1, 0, 64), (-1, 1, 64), (2, 1, 128), (3, 1, 128), (-1, 2, 128), (4, 2, 256), (5, 2, 256),
         (6, 2, 256), (7, 2, 256), (-1, 3, 256), (8, 3, 512), (9, 3, 512), (10, 3, 512), (11, 3, 512),
         (-1, 4, 512), (12, 4, 512), (13, 4, 512), (14, 4, 512), (15, 4, 512))
CONVS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 256), (256, 512),
         (512, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512), (512, 512))
SUPPORT = (-118, 133)  # conv5_4 feature i reads input rows [16 i - 118, 16 i + 133] (engine.VGG_SUPPORT)

# Bars, measured on an H100 80GB HBM3 (700 W limit); DESIGN.md 4.12 and 4.14.
# TAU_LAYER: |G - R| <= tau M of a bf16x3 launch against float64 on its own input (M = conv(|a|, |W|) + |b| forward,
#   conv_transpose(|g|, |W|) backward).  Set at 4x the worst of the first measurement, 9.9e-6 (conv1_1); over both
#   weight sets, noise and flat images at every shape of test_perceptual_gpu.LAUNCH_SHAPES the worst is 1.13e-5
#   forward (conv1_1, zero_bias) and 8.5e-6 backward (conv1_2), 3.5x under it.
# TAU_CHAIN: d(out) of every call (one window, tiles, pass splits, probe pairs) against the float64 chain of the GPU's
#   whole-image seed, |G - R| <= tau M element by element, M = chain(absolute=True): 4x the worst measured, 8.62e-6
#   in bf16x3 (biased, one window) and 1.38e-3 in bf16 (biased probe pair, tile 48 x 32).  Their ceilings, which any
#   real failure must clear: 20 x TAU_LAYER in bf16x3, 20 x the widest per-launch replay bar of bf16
#   (test_perceptual_bf16_cpu: acc_tau(512 x 9) + the 2^-8 of a bf16 store, in units of M).
TAU_LAYER = 4e-5
TAU_CHAIN = {"bf16x3": 3.5e-5, "bf16": 5.6e-3}
CHAIN_CEILING = {"bf16x3": 20 * TAU_LAYER, "bf16": 20 * ((512 * 9 // 16 + 2) * 2.0 ** -23 + 2.0 ** -8)}
BIAS_SPREAD = 1.0
ABS_LAUNCHES = 2  # chain(absolute=True): conv1_2's and conv1_1's data gradients in absolute values


# ------------------------------------------------------------------ weights
def state_dict(ws):
    """The PerceptualModel state dict of 16 (weight, bias) pairs (model.<index>.weight / .bias)."""
    sd, idx = {}, 0
    for conv, _, _ in STEPS:
        if conv >= 0:
            w, b = ws[conv]
            sd[f"model.{idx}.weight"], sd[f"model.{idx}.bias"] = w.clone(), b.clone()
            idx += 2  # Conv2d, ReLU
        else:
            idx += 1  # MaxPool2d
    return sd


@functools.lru_cache(maxsize=None)
def _zero_bias():
    from waternet_b200.training import PerceptualModel
    m = PerceptualModel(pretrained=False)
    convs = [c for c in m.model if isinstance(c, torch.nn.Conv2d)]
    return tuple((c.weight.detach().clone(), c.bias.detach().clone()) for c in convs)


@functools.lru_cache(maxsize=None)
def _biased(seed=17, h=64, w=64):
    """He-scaled weights; each layer's biases N(0, (BIAS_SPREAD sigma)^2), sigma the standard deviation of the
    layer's bias-free pre-activation on a noise image, evaluated layer by layer in float64 with the biases so far."""
    g = torch.Generator().manual_seed(seed)
    a = normalise(torch.rand(1, 3, h, w, generator=g, dtype=torch.float64))
    out = []
    for conv, _, _ in STEPS:
        if conv < 0:
            a = F.max_pool2d(a, 2, 2)
            continue
        cin, cout = CONVS[conv]
        wt = (torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5).float()
        z = F.conv2d(a, wt.double(), padding=1)
        b = (BIAS_SPREAD * z.std().item() * torch.randn(cout, generator=g)).float()
        a = F.relu(z + b.double().view(1, -1, 1, 1))
        out.append((wt, b))
    return tuple(out)


def weights(name):
    """16 (weight, bias) fp32 pairs of weight set ``name`` ("zero_bias" or "biased")."""
    return list({"zero_bias": _zero_bias, "biased": _biased}[name]())


WEIGHT_SETS = ("zero_bias", "biased")


def perceptual_model(name, precision="bf16x3", device="cuda"):
    """A native PerceptualModel carrying weight set ``name``."""
    from waternet_b200.training import PerceptualModel
    m = PerceptualModel(pretrained=False, native=True, precision=precision)
    m.load_state_dict(state_dict(weights(name)))
    return m.to(device).eval()


# ------------------------------------------------------------------ images
def normalise(x):
    """(x - mean) / std in float64, the constants as fp32 values."""
    mean = torch.tensor(MEAN, dtype=torch.float32).double().view(1, 3, 1, 1).to(x.device)
    return (x.double() - mean) / std64(x.device)


def std64(device):
    return torch.tensor(STD, dtype=torch.float32).double().view(1, 3, 1, 1).to(device)


def noise_pair(n, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = torch.rand((n, 3, h, w), generator=g)
    ref = (out + 0.3 * (torch.rand((n, 3, h, w), generator=g) - 0.5)).clamp(0, 1)
    return out, ref


FLAT_VALUES = (0.0, 1.0, 0.5, 0.8125)


def flat_pair(n, h, w, seed=0):
    """noise_pair with four flat patches per image in out (one value on all channels: 0, 1, 0.5, 0.8125), one of them
    at a corner of the image: the convolutions give equal values over a patch's interior, so the pools meet ties,
    positive ones wherever a channel's ReLU is on."""
    out, ref = noise_pair(n, h, w, seed)
    g = torch.Generator().manual_seed(seed + 1)
    ph, pw = max(8, h // 3), max(8, w // 3)
    for i in range(n):
        for k, v in enumerate(FLAT_VALUES):
            y = 0 if k == 0 else int(torch.randint(0, h - ph + 1, (1,), generator=g))
            x = 0 if k == 0 else int(torch.randint(0, w - pw + 1, (1,), generator=g))
            out[i, :, y:y + ph, x:x + pw] = v
    return out, ref


def pair(kind, n, h, w, seed=0):
    return {"noise": noise_pair, "flat": flat_pair}[kind](n, h, w, seed)


def probe_pair(n, h, w, patches, seed=0):
    """out uniform noise, ref == out except for 3 x 3 patches at (image, y, x) of ``patches``."""
    g = torch.Generator().manual_seed(seed)
    out = torch.rand((n, 3, h, w), generator=g)
    ref = out.clone()
    for i, y, x in patches:
        ref[i, :, y:y + 3, x:x + 3] = torch.rand((3, 3, 3), generator=g)
    return out, ref


# ------------------------------------------------------------------ references
def _conv_weight(ws, conv, device):
    return ws[conv][0].to(device, torch.float64)


def backward_launch(ws, fwd, gin, k, absolute=False):
    """float64 backward of forward launch k from its input gradient ``gin`` and the saved forward outputs ``fwd``
    (launch k - 1's output is launch k's input; launch 0's input has no ReLU).  A pool routes to the first maximum
    of each 2 x 2 window of its saved input (the floored edge gets 0); a convolution is conv_transpose with W, or with
    |W| when ``absolute`` (then ``gin`` is a magnitude), masked by ReLU' of its saved input."""
    conv = STEPS[k][0]
    if conv < 0:
        saved = fwd[k - 1]
        _, idx = F.max_pool2d(saved, 2, 2, return_indices=True)
        return F.max_unpool2d(gin, idx, 2, 2, output_size=saved.shape[-2:])
    w = _conv_weight(ws, conv, gin.device)
    r = F.conv_transpose2d(gin, w.abs() if absolute else w, padding=1)
    if k:
        r = r * (fwd[k - 1] > 0).double()
    return r


def backward_launch_reference(ws, fwd, gin, k):
    """(R, M) of backward launch k on its own input gradient ``gin``: M = conv_transpose(|g|, |W|) under the same
    ReLU' mask, None for a pool (exact)."""
    R = backward_launch(ws, fwd, gin, k)
    if STEPS[k][0] < 0:
        return R, None
    return R, backward_launch(ws, fwd, gin.abs(), k, absolute=True)


def chain(fwd, seed, ws, absolute=False):
    """d(loss)/d(out) in float64 from ``seed`` (d(loss)/d(conv5_4 before its ReLU)) through the 20 saved forward
    outputs ``fwd``.  ``absolute``: the magnitude M of each element instead -- the signed chain down to level 0, then
    the ABS_LAUNCHES launches of level 0 with |g| and |W| along the same masks.  (The whole chain in absolute values
    exceeds |R| by orders of magnitude -- 1e8 on the narrow VGG of test_perceptual_cpu, more at VGG's widths -- and
    a bar on it could not tell a dropped row from a right one; grad_reference.py makes the same choice.)"""
    g = seed.double()
    for k in range(len(STEPS) - 1, -1, -1):
        if absolute and k == ABS_LAUNCHES - 1:
            g = g.abs()
        g = backward_launch(ws, fwd, g, k, absolute and k < ABS_LAUNCHES)
    return g / std64(g.device)


def forward_outputs(x, ws):
    """The 20 forward launch outputs of x in float64 (bias, ReLU, first-maximum pools)."""
    a, outs = normalise(x), []
    for conv, _, _ in STEPS:
        if conv < 0:
            a = F.max_pool2d(a, 2, 2)
        else:
            w, b = ws[conv]
            a = F.relu(F.conv2d(a, w.to(a.device, torch.float64), b.to(a.device, torch.float64), padding=1))
        outs.append(a)
    return outs


def seed_of(fo, fr):
    """d(loss)/d(conv5_4 before its ReLU) of the loss from conv5_4 of out and ref."""
    return 2.0 * 255.0 ** 2 / fo.numel() * (fo.double() - fr.double()) * (fo > 0).double()


def support_mask(h, w, nonzero_features):
    """(n, 1, h, w) bool: the input pixels inside the support of some feature flagged in ``nonzero_features``
    ((n, h // 16, w // 16) bool); outside it every d(out) element is exactly 0."""
    dev = nonzero_features.device

    def rows(size, f):
        i = torch.arange(f, device=dev).view(-1, 1)
        y = torch.arange(size, device=dev).view(1, -1)
        return ((y >= 16 * i + SUPPORT[0]) & (y <= 16 * i + SUPPORT[1])).double()

    ry, rx = rows(h, nonzero_features.shape[1]), rows(w, nonzero_features.shape[2])
    cover = torch.einsum("iy,nij,jx->nyx", ry, nonzero_features.double(), rx)
    return (cover > 0).unsqueeze(1)


def assert_first_maximum_routing(device):
    """The pool references route a tie to the first maximum of its 2 x 2 window in row-major order, as the kernels
    do: torch's max_pool2d(return_indices=True) must pick that element on ``device``."""
    x = torch.tensor([[1.0, 1.0, 0.0, 2.0, 3.0, 1.0],
                      [1.0, 0.5, 2.0, 2.0, 0.0, 3.0],
                      [0.0, 0.0, 4.0, 4.0, 0.0, 0.5],
                      [0.0, 0.0, 4.0, 4.0, 0.5, 0.0]], dtype=torch.float64, device=device).view(1, 1, 4, 6)
    _, idx = F.max_pool2d(x, 2, 2, return_indices=True)
    want = torch.tensor([[0, 3, 4], [12, 14, 17]], device=device).view(1, 1, 2, 3)
    assert torch.equal(idx, want), idx
    g = torch.arange(1.0, 7.0, dtype=torch.float64, device=device).view(1, 1, 2, 3)
    routed = F.max_unpool2d(g, idx, 2, 2, output_size=(4, 6))
    assert routed.count_nonzero() == 6 and torch.equal(routed.view(-1)[want.view(-1)], g.view(-1))
