"""The native backward pass (wn_forward_train + wn_backward behind ``model(*ins)`` / ``out.backward(grad)``) against
float64 autograd, element by element (tests/grad_reference.py): the 34 parameter gradients and the 4 input-image
gradients, at shapes that reach every loop of the backward kernels -- degenerate images, widths and heights around
the 16 x 8 / 16 x 4 weight-gradient tiles and the 8 x 16 data-gradient tiles, several data-gradient tiles and
hundreds of weight-gradient tiles per CTA, tiles that span images -- on two networks whose ReLUs cannot flip."""
import gc

import numpy as np
import pytest
import torch

from grad_reference import (INPUT_NAMES, PARAM_NAMES, RELU_LAYERS, TAU, TAU_ONE_PIXEL, assert_grad_close,
                            assert_relus_cannot_flip, dead_channels, gated_state_dict, grad_error, reference,
                            smooth_state_dict)

pytestmark = pytest.mark.gpu

NETS = {"smooth": smooth_state_dict, "gated": gated_state_dict}
DENSE_SHAPES = [(3, 1, 1), (1, 1, 37), (1, 37, 1), (2, 3, 5),
                (1, 7, 15), (1, 9, 17), (1, 15, 16), (1, 17, 33),
                (4, 97, 131), (1, 385, 577), (300, 5, 7)]
PROBE_SHAPES = [(4, 97, 131), (1, 385, 577), (300, 5, 7)]
RADIUS = 13  # input-gradient support of one output pixel: the cmg kernels' radii 3+2+1+0+3+2+1+1 (refiners: 6)


def _shape_id(s):
    return "x".join(map(str, s))


@pytest.fixture(autouse=True)
def _free_device_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    gc.collect()
    torch.cuda.empty_cache()
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def _images(shape, seed):
    gen = torch.Generator().manual_seed(seed)
    return [torch.rand(shape[0], 3, shape[1], shape[2], generator=gen) for _ in range(4)]


def _native(sd, ins, grad, precision="default", prepare=None):
    """out, {param: grad}, [input grads] of one model(*ins) / out.backward(grad) on the library."""
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    leaves = [t.cuda().requires_grad_(True) for t in ins]
    used = prepare(leaves) if prepare else leaves
    out = m(*used)
    assert out.grad_fn is not None
    out.backward(grad.cuda().float())
    return out.detach(), {k: p.grad for k, p in m.named_parameters()}, [t.grad for t in leaves]


def _check(label, ref, params, inputs, keep=None, param_tau=TAU):
    """Every gradient against the reference: print the worst |G - R| / M per tensor, then assert it <= TAU
    (param_tau for the parameter gradients).  keep: optional (N,1,H,W) mask -- the input gradients are compared
    there only."""
    pairs = [(k, params[k], ref.grads[k], ref.M[k]) for k in PARAM_NAMES]
    for name, g, r, m in zip(INPUT_NAMES, inputs, ref.input_grads, ref.M_inputs):
        if keep is not None:
            g, r, m = g * keep, r * keep, m * keep
        pairs.append((name, g, r, m))
    worst = {name: grad_error(g, r, m).max().item() for name, g, r, m in pairs}
    print(f"\n{label}: worst |G - R| / M " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))
    for name, g, r, m in pairs:
        assert_grad_close(g, r, m, param_tau if name in ref.grads else TAU, f"{label} {name}")
    return worst


def _check_dead_channels_exactly_zero(params):
    """Channel-gated network: the rows of dead output channels and the columns of dead input channels are 0.0."""
    prev = None
    for layer in [f"cmg.conv{i}" for i in range(1, 9)]:
        w = params[layer + ".weight"]
        if layer in RELU_LAYERS:
            dead = dead_channels(layer)
            assert (w[dead] == 0).all() and (params[layer + ".bias"][dead] == 0).all(), layer
        if prev is not None:
            assert (w[:, dead_channels(prev)] == 0).all(), layer
        prev = layer
    for ref in ("wb_refiner", "ce_refiner", "gc_refiner"):
        for i in (1, 2, 3):
            layer = f"{ref}.conv{i}"
            dead = dead_channels(layer)
            assert (params[layer + ".weight"][dead] == 0).all() and (params[layer + ".bias"][dead] == 0).all(), layer
            if i > 1:
                assert (params[layer + ".weight"][:, dead_channels(f"{ref}.conv{i - 1}")] == 0).all(), layer


# ------------------------------------------------------------------ dense gradients
@pytest.mark.parametrize("shape", DENSE_SHAPES, ids=_shape_id)
@pytest.mark.parametrize("net", list(NETS))
def test_dense_gradients_match_fp64(net, shape):
    """MSE loss against a random target: every gradient element within TAU of its magnitude reference."""
    n, h, w = shape
    sd = NETS[net](21)
    ins = _images(shape, n * 7919 + h * 31 + w)
    target = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(h * w))
    ref = reference(sd, ins, target=target, device="cuda")
    assert_relus_cannot_flip(ref.z)
    out, params, inputs = _native(sd, ins, ref.seed.float())
    del ref.z
    assert (out.double() - ref.out).abs().max().item() <= 1e-3 * ref.out.abs().max().item()
    _check(f"dense {net} {_shape_id(shape)}", ref, params, inputs, param_tau=TAU_ONE_PIXEL if h * w == 1 else TAU)
    if net == "gated":
        _check_dead_channels_exactly_zero(params)


# ------------------------------------------------------------------ sparse probe gradients
def _probes(n, h, w, seed):
    """[(image, y, x)]: per image the corners and pixels on both sides of the weight-gradient seams (x = 16k-1 / 16k,
    y = 8k-1 / 8k, 4k-1 / 4k) and the data-gradient seams (x = 8k-1 / 8k, y = 16k-1 / 16k), greedily chosen more
    than 2 * RADIUS + 1 pixels apart.  Every third image of a batch of small images gets none."""
    rng = np.random.default_rng(seed)
    xs = sorted({v for k in range(1, w // 8 + 1) for v in (8 * k - 1, 8 * k) if v < w} | {0, w - 1})
    ys = sorted({v for k in range(1, h // 4 + 1) for v in (4 * k - 1, 4 * k) if v < h} | {0, h - 1})
    seams = [(y, x) for y in ys for x in xs]
    corners = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1)]
    probes = []
    for i in range(n):
        if n > 3 and i % 3 == 2 and i != n - 1:
            continue
        order = [seams[j] for j in rng.permutation(len(seams))]
        first = [(h - 1, w - 1)] if i == n - 1 else []
        mine = []
        for y, x in first + corners[i % 4:] + corners[:i % 4] + order:
            if all(max(abs(y - a), abs(x - b)) > 2 * RADIUS + 1 for a, b in mine):
                mine.append((y, x))
        probes += [(i, y, x) for y, x in mine]
    return probes


@pytest.mark.parametrize("shape", PROBE_SHAPES, ids=_shape_id)
@pytest.mark.parametrize("net", list(NETS))
def test_probe_gradients_stay_in_their_support(net, shape):
    """d(loss)/d(out) = +-1 at isolated pixels only: outside the radius-13 ball of every probe the input gradients
    are exactly 0.0 (nothing leaks into another pixel, tile or image); inside, and for the parameters, every element
    is within TAU of its magnitude reference."""
    n, h, w = shape
    sd = NETS[net](23)
    ins = _images(shape, 5 * n + h)
    probes = _probes(n, h, w, h * w)
    grad = torch.zeros(n, 3, h, w)
    keep = torch.zeros(n, 1, h, w, dtype=torch.bool)
    signs = torch.from_numpy(np.random.default_rng(n).choice([-1.0, 1.0], (len(probes), 3))).float()
    for (i, y, x), s in zip(probes, signs):
        grad[i, :, y, x] = s
        keep[i, :, max(0, y - RADIUS):y + RADIUS + 1, max(0, x - RADIUS):x + RADIUS + 1] = True
    assert len(probes) >= (n * 2 // 3 if n > 3 else 4 * n)
    ref = reference(sd, ins, grad=grad, device="cuda")
    assert_relus_cannot_flip(ref.z)
    del ref.z
    _, params, inputs = _native(sd, ins, grad)
    keep = keep.cuda()
    for name, g in zip(INPUT_NAMES, inputs):
        leak = g.masked_select(~keep.expand_as(g))
        assert (leak == 0).all(), f"{name}: {(leak != 0).sum().item()} nonzero input-gradient elements outside the probes' support"
    _check(f"probes {net} {_shape_id(shape)} ({len(probes)} probes)", ref, params, inputs, keep=keep.double())


# ------------------------------------------------------------------ same bits across modes and layouts
def test_precisions_and_input_layouts_give_the_same_bits():
    """The training forward always runs the bf16x3 scheme: precision "default" and "bf16x3" give identical outputs
    and gradients; so do channels-last inputs and views into larger images."""
    n, h, w = 2, 45, 70
    sd = gated_state_dict(25)
    ins = _images((n, h, w), 25)
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(26))
    base = _native(sd, ins, grad, "default")

    def same(other, label):
        assert torch.equal(other[0], base[0]), label
        for k in PARAM_NAMES:
            assert torch.equal(other[1][k], base[1][k]), f"{label}: {k}"
        for name, a, b in zip(INPUT_NAMES, other[2], base[2]):
            assert torch.equal(a, b), f"{label}: {name}"

    same(_native(sd, ins, grad, "bf16x3"), "bf16x3")
    same(_native(sd, ins, grad, "default", lambda ts: [t.contiguous(memory_format=torch.channels_last) for t in ts]),
         "channels_last")
    big = [torch.rand(n, 3, h + 6, w + 9, generator=torch.Generator().manual_seed(27)) for _ in range(4)]
    for b, t in zip(big, ins):
        b[:, :, 2:2 + h, 5:5 + w] = t
    out, params, inputs = _native(sd, big, grad, "default", lambda ts: [t[:, :, 2:2 + h, 5:5 + w] for t in ts])
    inner = [g[:, :, 2:2 + h, 5:5 + w].contiguous() for g in inputs]
    same((out, params, inner), "sliced views")
    for g in inputs:
        g[:, :, 2:2 + h, 5:5 + w] = 0
        assert (g == 0).all()


# ------------------------------------------------------------------ batch slices
def test_training_slices_match_fp64(monkeypatch):
    """A batch larger than the per-call pixel limit runs as slices whose parameter gradients are added: 3 slices
    against float64, not just against the one-call result."""
    from waternet_b200.engine import Engine
    n, h, w = 5, 24, 40
    monkeypatch.setattr(Engine, "TRAIN_MAX_PIXELS", 2 * h * w)   # slices of 2, 2, 1 images
    sd = gated_state_dict(29)
    ins = _images((n, h, w), 29)
    ref = reference(sd, ins, target=torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(30)), device="cuda")
    assert_relus_cannot_flip(ref.z)
    _, params, inputs = _native(sd, ins, ref.seed.float())
    _check("3 slices", ref, params, inputs)


def test_more_than_65535_images_train_as_two_slices():
    """70000 images of 1 x 1: one call may launch at most 65535 images (grid y), so the batch runs as two slices."""
    n = 70000
    sd = smooth_state_dict(31)
    ins = _images((n, 1, 1), 31)
    ref = reference(sd, ins, target=torch.rand(n, 3, 1, 1, generator=torch.Generator().manual_seed(32)), device="cuda")
    assert_relus_cannot_flip(ref.z)
    _, params, inputs = _native(sd, ins, ref.seed.float())
    _check("70000 x 1x1", ref, params, inputs, param_tau=TAU_ONE_PIXEL)


# ------------------------------------------------------------------ the reference itself
def test_gpu_reference_agrees_with_cpu_reference():
    sd = gated_state_dict(33)
    ins = _images((1, 37, 53), 33)
    grad = torch.randn(1, 3, 37, 53, generator=torch.Generator().manual_seed(34))
    cpu = reference(sd, ins, grad=grad)
    gpu = reference(sd, ins, grad=grad, device="cuda")

    def close(a, b, label):
        a = a.cpu()
        assert (a - b).abs().max().item() <= 1e-10 * b.abs().max().item(), label

    close(gpu.out, cpu.out, "out")
    for k in PARAM_NAMES:
        close(gpu.grads[k], cpu.grads[k], k)
        close(gpu.M[k], cpu.M[k], "M " + k)
    for i, name in enumerate(INPUT_NAMES):
        close(gpu.input_grads[i], cpu.input_grads[i], name)
        close(gpu.M_inputs[i], cpu.M_inputs[i], "M " + name)
    for k in RELU_LAYERS:
        close(gpu.z[k], cpu.z[k], "z " + k)
