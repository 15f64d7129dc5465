"""The windowed recompute backward of the sub-modules (``grad_tile`` on ``model.cmg``, the bound refiners and
free-standing ``ConfidenceMapGenerator`` / ``Refiner``: wn_confidence_maps_tiled / wn_refine_tiled +
wn_confidence_maps_backward_tiled / wn_refine_backward_tiled) against the untiled sub-module training call and against
float64 (``sub_reference`` of tests/test_submodule_train_gpu.py), element by element, on the two networks whose ReLUs
cannot flip: exactness when one window is one image, forward bits, dense gradients at tiles that put a pixel in one to
all windows, seam probes, bit reproducibility, isolation from the other stacks, a 12 Mpx image and the autograd
plumbing."""
import ctypes
import gc

import numpy as np
import pytest
import torch

from grad_reference import TAU, assert_grad_close, assert_relus_cannot_flip, gated_state_dict, smooth_state_dict
from test_submodule_train_gpu import _images, _sub, sub_reference
from test_submodule_train_gpu import _native as _reaches_library

pytestmark = pytest.mark.gpu

NETS = {"smooth": smooth_state_dict, "gated": gated_state_dict}
KINDS = ["cmg", "wb_refiner", "ce_refiner", "gc_refiner", "free_cmg", "free_refiner"]
PREFIX = {"free_cmg": "cmg", "free_refiner": "ce_refiner"}  # the state-dict entries a free-standing stack loads
RADIUS = {"cmg": 13, "refiner": 6}  # receptive-field radius of each stack


def _radius(prefix):
    return RADIUS["cmg" if prefix == "cmg" else "refiner"]


@pytest.fixture(autouse=True)
def _free_device_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _module(kind, sd, grad_tile=None):
    """(module to call, state-dict prefix of its parameters, the WaterNet it is bound to or None)."""
    from waternet_b200.net import ConfidenceMapGenerator, Refiner, WaterNet
    if kind.startswith("free_"):
        prefix = PREFIX[kind]
        m = ConfidenceMapGenerator() if prefix == "cmg" else Refiner()
        m.load_state_dict(_sub(sd, prefix))
        m.grad_tile = grad_tile
        return m.cuda(), prefix, None
    net = WaterNet(grad_tile=grad_tile)
    net.load_state_dict(sd)
    net = net.cuda().train()
    return getattr(net, kind), kind, net


def _call(mod, prefix, ins):
    if prefix == "cmg":
        return torch.cat(mod(*ins), 1)
    return mod(ins[0], ins[1])


def _run(kind, sd, ins, grad, grad_tile=None, prepare=None, wants=None):
    """out, {param: grad}, [input grads], the module and its parent after one call and out.backward(grad)."""
    mod, prefix, net = _module(kind, sd, grad_tile)
    n_in = 4 if prefix == "cmg" else 2
    wants = wants or [True] * n_in
    leaves = [t.cuda().requires_grad_(w) for t, w in zip(ins[:n_in], wants)]
    used = prepare(leaves) if prepare else leaves
    out = _call(mod, prefix, used)
    assert _reaches_library(out), "the call did not take the native training path"
    out.backward(grad.cuda())
    return out.detach(), {f"{prefix}.{k}": p.grad for k, p in mod.named_parameters()}, [t.grad for t in leaves], mod, net


def _same(a, b, label):
    assert torch.equal(a[0], b[0]), f"{label}: output"
    assert a[1].keys() == b[1].keys()
    for k in a[1]:
        assert torch.equal(a[1][k], b[1][k]), f"{label}: {k}"
    for i, (x, y) in enumerate(zip(a[2], b[2])):
        assert (x is None) == (y is None) and (x is None or torch.equal(x, y)), f"{label}: input {i}"


def _check(label, ref, grads, inputs, keep=None):
    worst = {}
    for k, r in ref.grads.items():
        worst[k] = assert_grad_close(grads[k], r, ref.M[k], TAU, f"{label} {k}")
    for i, (g, r, m) in enumerate(zip(inputs, ref.input_grads, ref.M_inputs)):
        if keep is not None:
            g, r, m = g * keep, r * keep, m * keep
        worst[f"input{i}"] = assert_grad_close(g, r, m, TAU, f"{label} input {i}")
    print(f"\n{label}: worst |G - R| / M {max(worst.values()):.2e}")


def _case(kind, net, shape, seed):
    sd = NETS[net](seed)
    prefix = PREFIX.get(kind, kind)
    n_in = 4 if prefix == "cmg" else 2
    ins = _images(shape, seed * 7 + shape[1], n_in)
    return sd, prefix, n_in, ins


# ------------------------------------------------------------------ exactness anchor and forward bits
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("net", list(NETS))
def test_one_window_per_image_equals_the_untiled_call(net, kind):
    """A tile at least as large as the image and one pass: every window is one image, the windowed call runs the
    untiled launches on the same data, and the output, the own-parameter and the input gradients agree bit for bit."""
    shape = (3, 45, 70)
    sd, _, _, ins = _case(kind, net, shape, 41)
    grad = torch.randn(*shape[:1], 3, *shape[1:], generator=torch.Generator().manual_seed(42))
    a = _run(kind, sd, ins, grad, grad_tile=(64, 96))
    b = _run(kind, sd, ins, grad)
    _same(a, b, f"{net} {kind} one window per image")


@pytest.mark.parametrize("shape,tile", [((1, 97, 131), 32), ((2, 5, 7), 1), ((3, 45, 70), (45, 16)),
                                        ((1, 385, 577), 128)])
@pytest.mark.parametrize("kind", ["cmg", "gc_refiner", "free_refiner"])
def test_forward_output_equals_the_untiled_training_forward(kind, shape, tile):
    sd, prefix, n_in, ins = _case(kind, "gated", shape, 43)
    leaves = [t.cuda().requires_grad_(True) for t in ins]
    tiled, untiled = _module(kind, sd, tile), _module(kind, sd)  # (module, prefix, parent): the parents stay alive
    a = _call(tiled[0], prefix, leaves)
    b = _call(untiled[0], prefix, leaves)
    assert _reaches_library(a) and _reaches_library(b) and torch.equal(a, b)


# ------------------------------------------------------------------ dense gradients against float64
DENSE = [((1, 97, 131), 32, 0), ((1, 97, 131), 8, 0), ((2, 5, 7), 1, 0), ((3, 45, 70), (45, 16), 0),
         ((2, 300, 500), 128, 5 * 126 * 151)]  # 24 windows of 126 x 151: passes of 5, 5, 5, 5, 4


def _dense_id(case):
    (n, h, w), tile, p = case
    return f"{n}x{h}x{w}-tile{tile if isinstance(tile, int) else '%dx%d' % tile}" + (f"-pass{p}" if p else "")


@pytest.mark.parametrize("case", DENSE, ids=_dense_id)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("net", list(NETS))
def test_dense_gradients_match_fp64(net, kind, case, monkeypatch):
    shape, tile, max_pass = case
    if max_pass:
        import waternet_b200.net as wnet
        monkeypatch.setattr(wnet, "TRAIN_PASS_PIXELS", max_pass)
    sd, prefix, _, ins = _case(kind, net, shape, 47)
    n, h, w = shape
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(h * w + n))
    ref = sub_reference(sd, prefix, ins, grad)
    assert_relus_cannot_flip(ref.z)
    out, grads, inputs, _, _ = _run(kind, sd, ins, grad, grad_tile=tile)
    assert (out.double() - ref.out).abs().max().item() <= 1e-3 * ref.out.abs().max().item()
    _check(f"dense {net} {kind} {_dense_id(case)}", ref, grads, inputs)


# ------------------------------------------------------------------ probes on seams
def _seam_probes(h, w, tile, radius, rng):
    """Pixels on both sides of every kept-rectangle boundary and at every window corner, greedily chosen more than
    2 * radius + 1 apart."""
    from waternet_b200.engine import tile_geometry
    g = tile_geometry(h, w, tile, tile)
    ys = {v for (r0, r1) in {win[2] for win in g["windows"]} for v in (r0, r0 - 1, r1 - 1, r1)}
    xs = {v for (c0, c1) in {win[3] for win in g["windows"]} for v in (c0, c0 - 1, c1 - 1, c1)}
    ys |= {v for y0 in {win[0] for win in g["windows"]} for v in (y0, y0 + g["win_h"] - 1)}
    xs |= {v for x0 in {win[1] for win in g["windows"]} for v in (x0, x0 + g["win_w"] - 1)}
    cand = [(y, x) for y in sorted(ys) for x in sorted(xs) if 0 <= y < h and 0 <= x < w]
    mine = []
    for k in rng.permutation(len(cand)):
        y, x = cand[k]
        if all(max(abs(y - a), abs(x - b)) > 2 * radius + 1 for a, b in mine):
            mine.append((y, x))
    return mine


@pytest.mark.parametrize("kind", ["cmg", "ce_refiner", "free_refiner"])
@pytest.mark.parametrize("net", list(NETS))
def test_probe_gradients_at_seams_stay_in_their_support(net, kind):
    n, h, w, tile = 2, 150, 190, 32
    sd, prefix, _, ins = _case(kind, net, (n, h, w), 53)
    radius = _radius(prefix)
    rng = np.random.default_rng(53)
    grad = torch.zeros(n, 3, h, w)
    keep = torch.zeros(n, 1, h, w, dtype=torch.bool)
    count = 0
    for i in range(n):
        for y, x in _seam_probes(h, w, tile, radius, rng):
            grad[i, :, y, x] = torch.from_numpy(rng.choice([-1.0, 1.0], 3)).float()
            keep[i, :, max(0, y - radius):y + radius + 1, max(0, x - radius):x + radius + 1] = True
            count += 1
    assert count >= 10
    ref = sub_reference(sd, prefix, ins, grad)
    assert_relus_cannot_flip(ref.z)
    _, grads, inputs, _, _ = _run(kind, sd, ins, grad, grad_tile=tile)
    keep = keep.cuda()
    for i, g in enumerate(inputs):
        leak = g.masked_select(~keep.expand_as(g))
        assert (leak == 0).all(), f"input {i}: {(leak != 0).sum().item()} nonzero elements outside the probes' support"
    _check(f"seam probes {net} {kind} ({count} probes)", ref, grads, inputs, keep=keep.double())


# ------------------------------------------------------------------ bits
def _abi_call(eng, prefix, which, ins, grad, shapes, tile, max_pass, fill=None):
    """wn_confidence_maps_backward_tiled / wn_refine_backward_tiled through the C ABI, the workspace optionally
    pre-filled with `fill` bytes.  Returns (own parameter gradients, input gradients)."""
    from waternet_b200 import _lib
    n, _, h, w = ins[0].shape
    stack = 0 if prefix == "cmg" else 1
    nbytes = eng.submodule_backward_tiled_workspace_bytes(n, h, w, stack, tile, max_pass)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    if fill is not None:
        ws.fill_(fill)
    first = 0 if stack == 0 else 16 + 6 * which
    grads = [torch.empty(tuple(s), device="cuda") for s in shapes]
    gin = [torch.empty(n, 3, h, w, device="cuda") for _ in ins]
    strides = (ctypes.c_int64 * (4 * len(ins)))(*[s for t in ins for s in t.stride()])
    arr = (ctypes.c_void_p * _lib.NUM_PARAMS)()
    for k, t in enumerate(grads):
        arr[first + k] = t.data_ptr()
    gin_arr = (ctypes.c_void_p * len(gin))(*[t.data_ptr() for t in gin])
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if stack == 0:
        rc = eng.lib.wn_confidence_maps_backward_tiled(eng.handle, *[t.data_ptr() for t in ins], strides,
                                                       grad.data_ptr(), arr, gin_arr, n, h, w, tile, tile, max_pass,
                                                       ws.data_ptr(), ws.numel(), stream)
    else:
        rc = eng.lib.wn_refine_backward_tiled(eng.handle, which, *[t.data_ptr() for t in ins], strides,
                                              grad.data_ptr(), arr, gin_arr, n, h, w, tile, tile, max_pass,
                                              ws.data_ptr(), ws.numel(), stream)
    _lib.check(rc, "sub-module backward tiled")
    torch.cuda.synchronize()
    return grads, gin


@pytest.mark.parametrize("kind", ["cmg", "gc_refiner"])
def test_same_bits_across_calls_workspaces_and_input_layouts(kind):
    n, h, w, tile = 2, 45, 70, 16
    sd, prefix, n_in, ins = _case(kind, "gated", (n, h, w), 59)
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(60))
    base = _run(kind, sd, ins, grad, grad_tile=tile)
    _same(_run(kind, sd, ins, grad, grad_tile=tile), base, "second call")
    _same(_run(kind, sd, ins, grad, grad_tile=tile,
               prepare=lambda ts: [t.contiguous(memory_format=torch.channels_last) for t in ts]), base, "channels_last")
    big = [torch.rand(n, 3, h + 6, w + 9, generator=torch.Generator().manual_seed(61)) for _ in range(n_in)]
    for b, t in zip(big, ins):
        b[:, :, 2:2 + h, 5:5 + w] = t
    out, grads, inputs, _, _ = _run(kind, sd, big, grad, grad_tile=tile,
                                    prepare=lambda ts: [t[:, :, 2:2 + h, 5:5 + w] for t in ts])
    _same((out, grads, [g[:, :, 2:2 + h, 5:5 + w].contiguous() for g in inputs]), base, "sliced views")

    mod, _, net = _module(kind, sd)
    eng = net.engine()
    shapes = [p.shape for p in mod.parameters()]
    dins = [t.cuda() for t in ins]
    which = None if prefix == "cmg" else mod._slot
    fresh = _abi_call(eng, prefix, which, dins, grad.cuda(), shapes, tile, 0)
    dirty = _abi_call(eng, prefix, which, dins, grad.cuda(), shapes, tile, 0, fill=0xFF)
    for a, b in zip(fresh[0] + fresh[1], dirty[0] + dirty[1]):
        assert torch.equal(a, b), "workspace pre-filled with 0xFF"
    for a, b in zip(fresh[0] + fresh[1], list(base[1].values()) + base[2]):
        assert torch.equal(a, b), "C ABI against the module"


@pytest.mark.parametrize("kind", ["cmg", "wb_refiner"])
def test_input_gradients_do_not_depend_on_the_pass_size(kind):
    n, h, w, tile = 2, 97, 131, 32  # 4 x 5 windows of 50 x 59 per image
    sd, prefix, _, ins = _case(kind, "gated", (n, h, w), 67)
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(68))
    ref = sub_reference(sd, prefix, ins, grad)
    mod, _, net = _module(kind, sd)
    eng = net.engine()
    shapes = [p.shape for p in mod.parameters()]
    dins = [t.cuda() for t in ins]
    which = None if prefix == "cmg" else mod._slot
    results = [_abi_call(eng, prefix, which, dins, grad.cuda(), shapes, tile, p)
               for p in (0, 3 * 50 * 59, 7 * 50 * 59)]
    names = list(ref.grads)
    for grads, gin in results:
        for a, b in zip(gin, results[0][1]):
            assert torch.equal(a, b)
        _check(f"pass size {kind}", ref, dict(zip(names, grads)), gin)


# ------------------------------------------------------------------ isolation
@pytest.mark.parametrize("kind", ["cmg", "wb_refiner", "ce_refiner", "gc_refiner"])
def test_bound_call_is_isolated_from_the_other_stacks(kind):
    """Other stacks' weights do not change a bound windowed call's bits, and their .grad stays None."""
    sd = smooth_state_dict(5)
    ins = _images((2, 37, 53), 11, 4)
    grad = torch.randn(2, 3, 37, 53, generator=torch.Generator().manual_seed(3))
    a = _run(kind, sd, ins, grad, grad_tile=16)
    scrambled = dict(sd)
    rng = torch.Generator().manual_seed(99)
    for k, v in sd.items():
        if not k.startswith(kind + "."):
            scrambled[k] = torch.randn(v.shape, generator=rng) * v.abs().max()
    b = _run(kind, scrambled, ins, grad, grad_tile=16)
    _same(a[:3], b[:3], f"{kind} with the other stacks scrambled")
    for net in (a[4], b[4]):
        for name, p in net.named_parameters():
            if not name.startswith(kind + "."):
                assert p.grad is None, name


# ------------------------------------------------------------------ beyond the untiled limit
@pytest.mark.parametrize("kind", ["cmg", "gc_refiner"])
def test_12_mpx_image_beyond_the_untiled_limit(kind):
    """1 x 3000 x 4000: over the untiled training call's limit (that call would evaluate the torch graph); the
    windowed one runs it in bounded memory, and its gradients agree with float64 references computed on crops of
    radius 2 * 13 around sparse probes."""
    from waternet_b200.engine import TRAIN_PASS_PIXELS, tile_geometry
    from waternet_b200 import _lib
    n, h, w, tile = 1, 3000, 4000, 998
    sd, prefix, n_in, _ = _case(kind, "smooth", (1, 8, 8), 71)
    ins = [t.cuda() for t in _images((n, h, w), 71, n_in)]
    untiled = _module(kind, sd)
    assert untiled[0]._train_engine(ins[0]) is None
    del untiled
    radius, crop = _radius(prefix), 2 * 13
    rng = np.random.default_rng(71)
    g = tile_geometry(h, w, tile, tile)
    cand = [(0, 0), (h - 1, w - 1), (0, w - 1), (h - 1, 0)]
    for y0, x0, (r0, r1), (c0, c1) in g["windows"]:
        cand += [(r0, c0), (r1 - 1, c1 - 1), (r0 - 1, c0), (y0, x0), (y0 + g["win_h"] - 1, x0 + g["win_w"] - 1)]
    cand += [(int(rng.integers(h)), int(rng.integers(w))) for _ in range(20)]
    probes = []
    for y, x in cand:
        if 0 <= y < h and 0 <= x < w and all(max(abs(y - a), abs(x - b)) > 2 * crop + 1 for a, b in probes):
            probes.append((y, x))
    probes = probes[:24]
    signs = rng.choice([-1.0, 1.0], (len(probes), 3))
    grad = torch.zeros(n, 3, h, w, device="cuda")
    for (y, x), s in zip(probes, signs):
        grad[0, :, y, x] = torch.from_numpy(s).float().cuda()

    mod, _, net = _module(kind, sd, tile)
    leaves = [t.requires_grad_(True) for t in ins]
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = _call(mod, prefix, leaves)
    out.backward(grad)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - held
    eng = net.engine()
    # the output, its copy through torch.cat for the cmg and its gradient, the input and the parameter gradients
    results = 3 * out.numel() * 4 + n_in * leaves[0].numel() * 4 + sum(p.numel() * 4 for p in mod.parameters())
    stack = 0 if prefix == "cmg" else 1
    budget = (eng.submodule_tiled_workspace_bytes(n, h, w, tile, _lib.MODE_BF16X3, max_pass_pixels=TRAIN_PASS_PIXELS)
              + eng.submodule_backward_tiled_workspace_bytes(n, h, w, stack, tile) + (1 << 30))
    print(f"\n{kind}: peak beyond inputs {peak / 2**30:.2f} GiB, results {results / 2**30:.2f} GiB, "
          f"budget {budget / 2**30:.2f} GiB")
    assert peak - results <= budget

    grads = {f"{prefix}.{k}": p.grad for k, p in mod.named_parameters()}
    inputs = [t.grad for t in leaves]
    keep = torch.zeros(n, 1, h, w, dtype=torch.bool, device="cuda")
    sums, msums = {}, {}
    for (y, x), s in zip(probes, signs):
        ya, yb, xa, xb = max(0, y - crop), min(h, y + crop + 1), max(0, x - crop), min(w, x + crop + 1)
        cg = torch.zeros(n, 3, yb - ya, xb - xa)
        cg[0, :, y - ya, x - xa] = torch.from_numpy(s).float()
        ref = sub_reference(sd, prefix, [t.detach()[:, :, ya:yb, xa:xb] for t in ins], cg)
        assert_relus_cannot_flip(ref.z)
        for k in ref.grads:
            sums[k] = sums.get(k, 0) + ref.grads[k]
            msums[k] = msums.get(k, 0) + ref.M[k]
        for i, (gi, r, mm) in enumerate(zip(inputs, ref.input_grads, ref.M_inputs)):
            assert_grad_close(gi[:, :, ya:yb, xa:xb], r, mm, TAU, f"12 Mpx {kind} probe ({y}, {x}) input {i}")
        keep[:, :, max(0, y - radius):y + radius + 1, max(0, x - radius):x + radius + 1] = True
    for i, gi in enumerate(inputs):
        assert (gi.masked_select(~keep.expand_as(gi)) == 0).all(), i
    for k in sums:
        assert_grad_close(grads[k], sums[k], msums[k], TAU, f"12 Mpx {kind} {k}")
    print(f"12 Mpx {kind}: {len(probes)} probes")


# ------------------------------------------------------------------ autograd plumbing
@pytest.mark.parametrize("kind", ["cmg", "ce_refiner", "free_cmg", "free_refiner"])
def test_autograd_plumbing(kind):
    n, h, w, tile = 1, 40, 60, 16
    sd, prefix, n_in, ins_cpu = _case(kind, "gated", (n, h, w), 73)
    ins = [t.cuda() for t in ins_cpu]
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(74)).cuda()
    base = _run(kind, sd, ins_cpu, grad.cpu(), grad_tile=tile)

    mod, _, parent = _module(kind, sd, tile)  #inputs only: the parameters do not require grad and get None
    for p in mod.parameters():
        p.requires_grad_(False)
    leaves = [t.clone().requires_grad_(True) for t in ins]
    _call(mod, prefix, leaves).backward(grad)
    assert all(p.grad is None for p in mod.parameters())
    for a, b in zip(leaves, base[2]):
        assert torch.equal(a.grad, b)

    mod, _, parent = _module(kind, sd, tile)  #parameters only
    out = _call(mod, prefix, ins)
    assert _reaches_library(out)
    out.backward(grad)
    for k, p in mod.named_parameters():
        assert torch.equal(p.grad, base[1][f"{prefix}.{k}"]), k

    mod, _, parent = _module(kind, sd, tile)  #some parameters frozen, one input alone
    mod.conv2.weight.requires_grad_(False)
    leaves = [t.clone().requires_grad_(i == n_in - 1) for i, t in enumerate(ins)]
    _call(mod, prefix, leaves).backward(grad)
    assert mod.conv2.weight.grad is None and torch.equal(mod.conv3.weight.grad, base[1][f"{prefix}.conv3.weight"])
    assert all(t.grad is None for t in leaves[:-1]) and torch.equal(leaves[-1].grad, base[2][-1])

    mod, _, parent = _module(kind, sd, tile)  #an input edited in place between forward and backward
    leaf = ins[0].clone().requires_grad_(True)
    x = leaf * 1.0
    out = _call(mod, prefix, [x] + ins[1:])
    x.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.backward(grad)

    mod, _, parent = _module(kind, sd, tile)  #parameters modified between forward and backward
    out = _call(mod, prefix, ins)
    with torch.no_grad():
        mod.conv1.weight.mul_(1.5)
    _call(mod, prefix, [t[:, :, :8, :8] for t in ins])  # repacks the changed weights
    with pytest.raises(RuntimeError, match="modified between forward and backward"):
        out.backward(grad)
