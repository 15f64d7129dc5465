"""The sub-modules under autograd (``model.cmg(...)``, ``model.wb_refiner(...)``, free-standing
``ConfidenceMapGenerator`` / ``Refiner`` with parameters or inputs that require grad): the native training path
(wn_confidence_maps_train / _backward, wn_refine_train / _backward) against float64 autograd through
``oracle/forward.py``, element by element with the bar of tests/grad_reference.py; isolation from the rest of the
network; partial requires_grad, layouts and precisions; batch slices; and a short training loop."""
import copy
import ctypes
import gc
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from grad_reference import (RELU_LAYERS, TAU, TAU_ONE_PIXEL, _leaves, assert_grad_close, assert_relus_cannot_flip,
                            gated_state_dict, smooth_state_dict)
from oracle import forward as ofw

pytestmark = pytest.mark.gpu

NETS = {"smooth": smooth_state_dict, "gated": gated_state_dict}
# 1 x 1 images, odd sizes, several images, data-gradient (8 x 16) and weight-gradient (16 x 8 / 16 x 4) tile seams
SHAPES = [(3, 1, 1), (2, 3, 5), (1, 17, 33), (2, 37, 53), (1, 97, 131)]
KINDS = ["cmg", "wb_refiner", "ce_refiner", "gc_refiner", "free_cmg", "free_refiner"]
PREFIX = {"free_cmg": "cmg", "free_refiner": "ce_refiner"}  # the state-dict entries a free-standing stack loads


def _shape_id(s):
    return "x".join(map(str, s))


@pytest.fixture(autouse=True)
def _free_device_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _images(shape, seed, count):
    gen = torch.Generator().manual_seed(seed)
    return [torch.rand(shape[0], 3, shape[1], shape[2], generator=gen) for _ in range(count)]


def _sub(sd, prefix):
    return {k[len(prefix) + 1:]: v for k, v in sd.items() if k.startswith(prefix + ".")}


def _module(kind, sd, precision="default"):
    """(module to call, state-dict prefix of its parameters, the WaterNet it is bound to or None)."""
    from waternet_b200.net import ConfidenceMapGenerator, Refiner, WaterNet
    if kind == "free_cmg":
        m = ConfidenceMapGenerator()
        m.load_state_dict(_sub(sd, "cmg"))
        m.precision = precision
        return m.cuda(), "cmg", None
    if kind == "free_refiner":
        m = Refiner()
        m.load_state_dict(_sub(sd, "ce_refiner"))
        m.precision = precision
        return m.cuda(), "ce_refiner", None
    net = WaterNet(precision=precision)
    net.load_state_dict(sd)
    net = net.cuda().train()
    return getattr(net, kind), kind, net


def _call(mod, prefix, ins):
    """The sub-module's output as one (N,3,H,W) tensor.  A refiner reads (x, ins[1])."""
    if prefix == "cmg":
        return torch.cat(mod(*ins), 1)
    return mod(ins[0], ins[1])


def _native(out, depth=4):
    """The autograd graph of ``out`` reaches the library's sub-module node within ``depth`` steps."""
    front = [out.grad_fn]
    for _ in range(depth):
        if any(f is not None and "SubmoduleForward" in type(f).__name__ for f in front):
            return True
        front = [g for f in front if f is not None for g, _ in f.next_functions]
    return False


def _own_grads(mod, prefix):
    return {f"{prefix}.{k}": p.grad for k, p in mod.named_parameters()}


def sub_reference(sd, prefix, ins, grad, device="cuda"):
    """Float64 output and gradients of the sub-module ``prefix`` ("cmg" or a refiner) of the network state dict
    ``sd`` at its inputs ``ins`` (4 images for the cmg, (x, xbar) for a refiner), back-propagating ``grad``.  The
    magnitude reference M is that of grad_reference.reference, for this stack alone: every convolution fed its
    reference input in absolute values, with |W|, |b|, weighted by the absolute value of its output gradient."""
    layers = ofw.CMG_LAYERS if prefix == "cmg" else ofw.REFINER_LAYERS
    keys = [f"{prefix}.{name}.{p}" for name, _, _, _ in layers for p in ("weight", "bias")]
    params = dict(zip(keys, _leaves([sd[k] for k in keys], device)))
    leaves = _leaves(ins, device)
    seen = {}
    t = torch.cat(leaves, 1)
    for name, _, _, k in layers:
        layer = f"{prefix}.{name}"
        z = F.conv2d(t, params[layer + ".weight"], params[layer + ".bias"], padding=k // 2)
        z.retain_grad()
        seen[layer] = (t, z, k)
        t = torch.sigmoid(z) if layer == "cmg.conv8" else F.relu(z)
    t.backward(grad.detach().to(device, torch.float64))
    res = types.SimpleNamespace(out=t.detach(), grads={k: v.grad for k, v in params.items()},
                                input_grads=[v.grad for v in leaves],
                                z={k: z.detach() for k, (_, z, _) in seen.items() if k in RELU_LAYERS})
    pabs = dict(zip(keys, _leaves([sd[k] for k in keys], device, absolute=True)))
    labs = _leaves(ins, device, absolute=True)
    total = 0
    for i, (layer, (a, z, k)) in enumerate(seen.items()):
        a = torch.cat(labs, 1) if i == 0 else a.detach().abs()
        total = total + (F.conv2d(a, pabs[layer + ".weight"], pabs[layer + ".bias"], padding=k // 2)
                         * z.grad.abs()).sum()
    total.backward()
    res.M = {k: v.grad for k, v in pabs.items()}
    res.M_inputs = [v.grad for v in labs]
    return res


def _run(kind, sd, ins, grad, precision="default", prepare=None, wants=None):
    """out, {param: grad}, [input grads], the module and its parent after one call and out.backward(grad)."""
    mod, prefix, net = _module(kind, sd, precision)
    n_in = 4 if prefix == "cmg" else 2
    wants = wants or [True] * n_in
    leaves = [t.cuda().requires_grad_(w) for t, w in zip(ins[:n_in], wants)]
    used = prepare(leaves) if prepare else leaves
    out = _call(mod, prefix, used)
    assert _native(out), "the call did not take the native training path"
    out.backward(grad.cuda())
    return out.detach(), _own_grads(mod, prefix), [t.grad for t in leaves], mod, net


def _check(label, ref, grads, inputs, param_tau):
    worst = {}
    for k, r in ref.grads.items():
        worst[k] = assert_grad_close(grads[k], r, ref.M[k], param_tau, f"{label} {k}")
    for i, (g, r, m) in enumerate(zip(inputs, ref.input_grads, ref.M_inputs)):
        worst[f"input{i}"] = assert_grad_close(g, r, m, TAU, f"{label} input {i}")
    print(f"\n{label}: worst |G - R| / M " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


# ------------------------------------------------------------------ float64 agreement
@pytest.mark.parametrize("shape", SHAPES, ids=_shape_id)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("net", list(NETS))
def test_gradients_match_fp64(net, kind, shape):
    n, h, w = shape
    sd = NETS[net](31)
    prefix = PREFIX.get(kind, kind)
    n_in = 4 if prefix == "cmg" else 2
    ins = _images(shape, n * 7919 + h * 31 + w + len(kind), n_in)
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(h * w + n))
    ref = sub_reference(sd, prefix, ins, grad)
    assert_relus_cannot_flip(ref.z)
    out, grads, inputs, _, _ = _run(kind, sd, ins, grad)
    assert (out.double() - ref.out).abs().max().item() <= 1e-3 * ref.out.abs().max().item()
    _check(f"{net} {kind} {_shape_id(shape)}", ref, grads, inputs, TAU_ONE_PIXEL if h * w == 1 else TAU)


# ------------------------------------------------------------------ isolation
@pytest.mark.parametrize("kind", ["cmg", "wb_refiner", "ce_refiner", "gc_refiner"])
def test_bound_call_is_isolated_from_the_other_stacks(kind):
    """Other stacks' weights do not change a bound call's bits, and their .grad stays None."""
    sd = smooth_state_dict(5)
    ins = _images((2, 37, 53), 11, 4)
    grad = torch.randn(2, 3, 37, 53, generator=torch.Generator().manual_seed(3))
    out_a, grads_a, in_a, _, net_a = _run(kind, sd, ins, grad)
    scrambled = dict(sd)
    rng = torch.Generator().manual_seed(99)
    for k, v in sd.items():
        if not k.startswith(kind + "."):
            scrambled[k] = torch.randn(v.shape, generator=rng) * v.abs().max()
    out_b, grads_b, in_b, _, net_b = _run(kind, scrambled, ins, grad)
    assert torch.equal(out_a, out_b)
    for k in grads_a:
        assert torch.equal(grads_a[k], grads_b[k]), k
    for a, b in zip(in_a, in_b):
        assert torch.equal(a, b)
    for net in (net_a, net_b):
        for name, p in net.named_parameters():
            if not name.startswith(kind + "."):
                assert p.grad is None, name


# ------------------------------------------------------------------ partial requires_grad, layouts, precisions
@pytest.mark.parametrize("kind", ["cmg", "gc_refiner", "free_refiner"])
def test_partial_requires_grad_layouts_and_precisions_give_the_same_bits(kind):
    sd = smooth_state_dict(8)
    prefix = PREFIX.get(kind, kind)
    n_in = 4 if prefix == "cmg" else 2
    ins = _images((3, 21, 40), 4, n_in)
    grad = torch.randn(3, 3, 21, 40, generator=torch.Generator().manual_seed(8))
    out, grads, inputs, _, _ = _run(kind, sd, ins, grad)
    variants = {
        "bf16x3": dict(precision="bf16x3"),
        "channels_last": dict(prepare=lambda ls: [t.contiguous(memory_format=torch.channels_last) for t in ls]),
        "sliced": dict(prepare=lambda ls: [torch.cat([t, t], 3)[:, :, :, 40:] for t in ls]),
    }
    for name, kw in variants.items():
        o, g, i, _, _ = _run(kind, sd, ins, grad, **kw)
        assert torch.equal(o, out), name
        assert all(torch.equal(g[k], grads[k]) for k in grads), name
        assert all(torch.equal(a, b) for a, b in zip(i, inputs)), name
    for only in range(n_in):  # one input alone
        wants = [j == only for j in range(n_in)]
        o, g, i, _, _ = _run(kind, sd, ins, grad, wants=wants)
        assert torch.equal(o, out) and torch.equal(i[only], inputs[only])
        assert all(t is None for j, t in enumerate(i) if j != only)
        assert all(torch.equal(g[k], grads[k]) for k in grads)
    # parameters only
    o, g, i, _, _ = _run(kind, sd, ins, grad, wants=[False] * n_in)
    assert torch.equal(o, out) and all(t is None for t in i)
    assert all(torch.equal(g[k], grads[k]) for k in grads)
    # inputs only: no parameter gradient
    mod, _, _ = _module(kind, sd)
    for p in mod.parameters():
        p.requires_grad_(False)
    leaves = [t.cuda().requires_grad_(True) for t in ins]
    _call(mod, prefix, leaves).backward(grad.cuda())
    assert all(p.grad is None for p in mod.parameters())
    assert all(torch.equal(a.grad, b) for a, b in zip(leaves, inputs))


def test_eight_bit_levels_take_the_exact_first_layer_and_match_fp64():
    """Inputs that are 8-bit levels (u / 255) drop the first layer's a_lo pass, as wn_forward_train does."""
    sd = smooth_state_dict(12)
    ins = [torch.from_numpy(ofw.synthetic_image(i, 33, 47, "smooth")).permute(2, 0, 1)[None].float() / 255
           for i in range(4)]
    grad = torch.randn(1, 3, 33, 47, generator=torch.Generator().manual_seed(1))
    for kind in ("cmg", "ce_refiner"):
        prefix = kind
        n_in = 4 if prefix == "cmg" else 2
        ref = sub_reference(sd, prefix, ins[:n_in], grad)
        out, grads, inputs, _, _ = _run(kind, sd, ins, grad)
        assert (out.double() - ref.out).abs().max().item() <= 1e-3 * ref.out.abs().max().item()
        _check(f"levels {kind}", ref, grads, inputs, TAU)


# ------------------------------------------------------------------ batch slices
@pytest.mark.parametrize("kind", ["cmg", "wb_refiner", "free_refiner"])
def test_batch_slices_match_fp64(kind, monkeypatch):
    from waternet_b200.engine import Engine
    n, h, w = 5, 19, 24
    monkeypatch.setattr(Engine, "TRAIN_MAX_PIXELS", 2 * h * w)  # slices of 2, 2 and 1 images
    sd = smooth_state_dict(17)
    prefix = PREFIX.get(kind, kind)
    ins = _images((n, h, w), 23, 4 if prefix == "cmg" else 2)
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(5))
    ref = sub_reference(sd, prefix, ins, grad)
    out, grads, inputs, _, _ = _run(kind, sd, ins, grad)
    assert (out.double() - ref.out).abs().max().item() <= 1e-3 * ref.out.abs().max().item()
    _check(f"slices {kind}", ref, grads, inputs, TAU)


# ------------------------------------------------------------------ errors
def test_parameters_changed_between_forward_and_backward_raise():
    sd = smooth_state_dict(2)
    ins = [t.cuda() for t in _images((1, 16, 16), 2, 4)]
    for kind in ("cmg", "ce_refiner", "free_cmg", "free_refiner"):
        mod, prefix, _ = _module(kind, sd)
        out = _call(mod, prefix, ins)
        with torch.no_grad():
            mod.conv1.weight.mul_(1.5)
        _call(mod, prefix, [t[:, :, :8, :8] for t in ins])  # repacks the changed weights
        with pytest.raises(RuntimeError, match="modified between forward and backward"):
            out.sum().backward()


def test_calls_without_packed_weights_are_refused():
    from waternet_b200 import _lib
    from waternet_b200.engine import new_engine
    eng = new_engine("cuda:0")
    buf = torch.zeros(4096, device="cuda")
    p = buf.data_ptr()
    strides = (ctypes.c_int64 * 16)(*([768, 256, 16, 1] * 4))
    grads = (ctypes.c_void_p * _lib.NUM_PARAMS)(*([p] * _lib.NUM_PARAMS))
    lib, h = eng.lib, eng.handle
    assert lib.wn_confidence_maps_train(h, p, p, p, p, strides, p, 1, 16, 16, p, 1 << 30, None) == -3
    assert lib.wn_confidence_maps_backward(h, p, grads, None, 1, 16, 16, p, 1 << 30, None) == -3
    assert lib.wn_refine_train(h, 0, p, p, strides, p, 1, 16, 16, p, 1 << 30, None) == -3
    assert lib.wn_refine_backward(h, 2, p, grads, None, 1, 16, 16, p, 1 << 30, None) == -3
    assert b"wn_pack_weights" in lib.wn_last_error()


def test_a_too_small_workspace_is_refused():
    from waternet_b200 import _lib
    m = _module("wb_refiner", smooth_state_dict(3))[2]
    eng = m.engine()
    need = eng.lib.wn_submodule_train_workspace_bytes(1, 16, 16, 1)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    x, out = torch.rand(1, 3, 16, 16, device="cuda"), torch.empty(1, 3, 16, 16, device="cuda")
    strides = (ctypes.c_int64 * 8)(*(list(x.stride()) * 2))
    args = (eng.handle, 0, x.data_ptr(), x.data_ptr(), strides, out.data_ptr(), 1, 16, 16, ws.data_ptr())
    assert eng.lib.wn_refine_train(*args, need - 1, None) == -4
    assert eng.lib.wn_refine_train(*args, need, None) == 0
    # the inference call, whose first layer is the fused one: kRL1 gives each channel the same sums
    assert torch.equal(out, eng.refine(0, x, x, _lib.MODE_BF16X3))


# ------------------------------------------------------------------ training loop
@pytest.mark.parametrize("kind", ["cmg", "gc_refiner"])
def test_native_training_steps_track_the_torch_graph(kind):
    """20 Adam steps of one sub-module with native gradients follow the loss curve of torch autograd (TF32 off)."""
    from waternet_b200.net import WaterNet
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        net = WaterNet()
        net.load_state_dict(ofw.synthetic_state_dict(6, 1.0))
        net = net.cuda().train()
        twin = copy.deepcopy(net)
        ins = [t.cuda() for t in _images((4, 32, 32), 40, 4)]
        target = torch.rand(4, 3, 32, 32, generator=torch.Generator().manual_seed(41)).cuda()
        mod_a, mod_b = getattr(net, kind), getattr(twin, kind)
        opt_a = torch.optim.Adam(mod_a.parameters(), lr=1e-3)
        opt_b = torch.optim.Adam(mod_b.parameters(), lr=1e-3)
        la, lb = [], []
        for _ in range(20):
            for mod, opt, losses, native in ((mod_a, opt_a, la, True), (mod_b, opt_b, lb, False)):
                opt.zero_grad()
                if kind == "cmg":
                    out = torch.cat(mod(*ins), 1) if native else mod._graph(*ins)
                else:
                    out = mod(ins[0], ins[3]) if native else mod._graph(ins[0], ins[3])
                loss = F.mse_loss(out, target)
                loss.backward()
                opt.step()
                losses.append(loss.item())
        assert la[-1] < la[0]
        assert np.allclose(la, lb, rtol=2e-3), (la, lb)
        assert all(p.grad is None for p in net.wb_refiner.parameters())
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
