"""The windowed recompute backward (``WaterNet.grad_tile``: wn_forward_tiled + wn_backward_tiled) against the untiled
native backward and against float64 (tests/grad_reference.py), element by element, on the two networks whose ReLUs
cannot flip: exactness when one window is one image, dense gradients at tiles that put a pixel in one to all windows,
probes on kept-rectangle seams and window corners, bit reproducibility, a 12 Mpx image that the untiled path refuses,
and the autograd plumbing."""
import ctypes
import gc

import numpy as np
import pytest
import torch

from grad_reference import (INPUT_NAMES, PARAM_NAMES, TAU, assert_grad_close, assert_relus_cannot_flip,
                            gated_state_dict, grad_error, reference, smooth_state_dict)

pytestmark = pytest.mark.gpu

NETS = {"smooth": smooth_state_dict, "gated": gated_state_dict}
RADIUS = 13


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


def _model(sd, grad_tile=None):
    from waternet_b200.net import WaterNet
    m = WaterNet(grad_tile=grad_tile)
    m.load_state_dict(sd, strict=True)
    return m.cuda().train()


def _native(sd, ins, grad, grad_tile=None, prepare=None):
    """out, {param: grad}, [input grads] of one model(*ins) / out.backward(grad)."""
    m = _model(sd, grad_tile)
    leaves = [t.cuda().requires_grad_(True) for t in ins]
    used = prepare(leaves) if prepare else leaves
    out = m(*used)
    assert out.grad_fn is not None
    out.backward(grad.cuda().float())
    return out.detach(), {k: p.grad for k, p in m.named_parameters()}, [t.grad for t in leaves]


def _check(label, ref, params, inputs, keep=None):
    pairs = [(k, params[k], ref.grads[k], ref.M[k]) for k in PARAM_NAMES]
    for name, g, r, m in zip(INPUT_NAMES, inputs, ref.input_grads, ref.M_inputs):
        if keep is not None:
            g, r, m = g * keep, r * keep, m * keep
        pairs.append((name, g, r, m))
    worst = max(grad_error(g, r, m).max().item() for _, g, r, m in pairs)
    print(f"\n{label}: worst |G - R| / M {worst:.2e}")
    for name, g, r, m in pairs:
        assert_grad_close(g, r, m, TAU, f"{label} {name}")


def _same(a, b, label):
    assert torch.equal(a[0], b[0]), f"{label}: output"
    for k in PARAM_NAMES:
        assert torch.equal(a[1][k], b[1][k]), f"{label}: {k}"
    for name, x, y in zip(INPUT_NAMES, a[2], b[2]):
        assert torch.equal(x, y), f"{label}: {name}"


# ------------------------------------------------------------------ exactness anchor and forward bits
@pytest.mark.parametrize("net", list(NETS))
def test_one_window_per_image_equals_the_untiled_backward(net):
    """A tile at least as large as the image and one pass for the batch: every window is one image, the windowed
    call runs the untiled launches on the same data, and every output and gradient bit agrees."""
    n, h, w = 3, 45, 70
    sd = NETS[net](41)
    ins = _images((n, h, w), 41)
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(42))
    _same(_native(sd, ins, grad, grad_tile=(64, 96)), _native(sd, ins, grad), "one window per image")


@pytest.mark.parametrize("shape,tile", [((1, 97, 131), 32), ((2, 5, 7), 1), ((3, 45, 70), (45, 16)),
                                        ((1, 385, 577), 128)])
def test_forward_output_equals_the_untiled_training_forward(shape, tile):
    sd = gated_state_dict(43)
    ins = [t.cuda().requires_grad_(True) for t in _images(shape, 43)]
    a = _model(sd, tile)(*ins)
    b = _model(sd)(*ins)
    assert a.grad_fn is not None and torch.equal(a, b)


# ------------------------------------------------------------------ dense gradients against float64
DENSE = [((1, 97, 131), 32, 0), ((1, 97, 131), 8, 0), ((2, 5, 7), 1, 0), ((3, 45, 70), (45, 16), 0),
         ((2, 300, 500), 128, 5 * 126 * 151)]  # 24 windows of 126 x 151: passes of 5, 5, 5, 5, 4


def _dense_id(case):
    (n, h, w), tile, p = case
    return f"{n}x{h}x{w}-tile{tile if isinstance(tile, int) else '%dx%d' % tile}" + (f"-pass{p}" if p else "")


@pytest.mark.parametrize("case", DENSE, ids=_dense_id)
@pytest.mark.parametrize("net", list(NETS))
def test_dense_gradients_match_fp64(net, case, monkeypatch):
    (n, h, w), tile, max_pass = case
    if max_pass:
        import waternet_b200.net as wnet
        monkeypatch.setattr(wnet, "TRAIN_PASS_PIXELS", max_pass)
    sd = NETS[net](47)
    ins = _images((n, h, w), n * 31 + h)
    target = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(h * w))
    ref = reference(sd, ins, target=target, device="cuda")
    assert_relus_cannot_flip(ref.z)
    del ref.z
    out, params, inputs = _native(sd, ins, ref.seed.float(), grad_tile=tile)
    assert (out.double() - ref.out).abs().max().item() <= 1e-3 * ref.out.abs().max().item()
    _check(f"dense {net} {_dense_id(case)}", ref, params, inputs)
    if net == "gated":
        from test_backward_gpu import _check_dead_channels_exactly_zero
        _check_dead_channels_exactly_zero(params)


# ------------------------------------------------------------------ probes on seams
def _seam_probes(h, w, tile, rng):
    """Pixels on both sides of every kept-rectangle boundary and at every window corner, greedily chosen more than
    2 * RADIUS + 1 apart."""
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
        if all(max(abs(y - a), abs(x - b)) > 2 * RADIUS + 1 for a, b in mine):
            mine.append((y, x))
    return mine


@pytest.mark.parametrize("net", list(NETS))
def test_probe_gradients_at_seams_stay_in_their_support(net):
    n, h, w, tile = 2, 150, 190, 32
    sd = NETS[net](53)
    ins = _images((n, h, w), 53)
    rng = np.random.default_rng(53)
    grad = torch.zeros(n, 3, h, w)
    keep = torch.zeros(n, 1, h, w, dtype=torch.bool)
    count = 0
    for i in range(n):
        for y, x in _seam_probes(h, w, tile, rng):
            grad[i, :, y, x] = torch.from_numpy(rng.choice([-1.0, 1.0], 3)).float()
            keep[i, :, max(0, y - RADIUS):y + RADIUS + 1, max(0, x - RADIUS):x + RADIUS + 1] = True
            count += 1
    assert count >= 10
    ref = reference(sd, ins, grad=grad, device="cuda")
    assert_relus_cannot_flip(ref.z)
    del ref.z
    _, params, inputs = _native(sd, ins, grad, grad_tile=tile)
    keep = keep.cuda()
    for name, g in zip(INPUT_NAMES, inputs):
        leak = g.masked_select(~keep.expand_as(g))
        assert (leak == 0).all(), f"{name}: {(leak != 0).sum().item()} nonzero input-gradient elements outside the probes' support"
    _check(f"seam probes {net} ({count} probes)", ref, params, inputs, keep=keep.double())


# ------------------------------------------------------------------ bits
def _abi_call(eng, ins, grad, shapes, tile, max_pass, fill=None):
    """wn_backward_tiled through the C ABI, with the workspace optionally pre-filled with `fill` bytes."""
    from waternet_b200 import _lib
    n, _, h, w = ins[0].shape
    nbytes = eng.backward_tiled_workspace_bytes(n, h, w, tile, max_pass)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    if fill is not None:
        ws.fill_(fill)
    grads = [torch.empty(tuple(s), device="cuda") for s in shapes]
    gin = [torch.empty(n, 3, h, w, device="cuda") for _ in range(4)]
    strides = (ctypes.c_int64 * 16)(*[s for t in ins for s in t.stride()])
    arr = (ctypes.c_void_p * _lib.NUM_PARAMS)(*[t.data_ptr() for t in grads])
    gin_arr = (ctypes.c_void_p * 4)(*[t.data_ptr() for t in gin])
    rc = eng.lib.wn_backward_tiled(eng.handle, *[t.data_ptr() for t in ins], strides, grad.data_ptr(), arr, gin_arr,
                                   n, h, w, tile, tile, max_pass, ws.data_ptr(), ws.numel(),
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, "wn_backward_tiled")
    torch.cuda.synchronize()
    return grads, gin


def test_same_bits_across_calls_workspaces_and_input_layouts():
    n, h, w, tile = 2, 45, 70, 16
    sd = gated_state_dict(59)
    ins = _images((n, h, w), 59)
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(60))
    base = _native(sd, ins, grad, grad_tile=tile)
    _same(_native(sd, ins, grad, grad_tile=tile), base, "second call")
    _same(_native(sd, ins, grad, grad_tile=tile,
                  prepare=lambda ts: [t.contiguous(memory_format=torch.channels_last) for t in ts]), base,
          "channels_last")
    big = [torch.rand(n, 3, h + 6, w + 9, generator=torch.Generator().manual_seed(61)) for _ in range(4)]
    for b, t in zip(big, ins):
        b[:, :, 2:2 + h, 5:5 + w] = t
    out, params, inputs = _native(sd, big, grad, grad_tile=tile, prepare=lambda ts: [t[:, :, 2:2 + h, 5:5 + w] for t in ts])
    _same((out, params, [g[:, :, 2:2 + h, 5:5 + w].contiguous() for g in inputs]), base, "sliced views")

    m = _model(sd)
    eng = m.engine()
    shapes = [p.shape for p in m._ordered_params()]
    dins = [t.cuda() for t in ins]
    dgrad = grad.cuda()
    fresh = _abi_call(eng, dins, dgrad, shapes, tile, 0)
    dirty = _abi_call(eng, dins, dgrad, shapes, tile, 0, fill=0xFF)
    for a, b in zip(fresh[0] + fresh[1], dirty[0] + dirty[1]):
        assert torch.equal(a, b), "workspace pre-filled with 0xFF"
    for a, b in zip(fresh[0] + fresh[1], list(base[1].values()) + base[2]):
        assert torch.equal(a, b), "C ABI against the model"


def test_input_gradients_do_not_depend_on_the_pass_size():
    n, h, w, tile = 2, 97, 131, 32  # 4 x 5 windows of 50 x 59 per image
    sd = gated_state_dict(67)
    ins = _images((n, h, w), 67)
    target = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(68))
    ref = reference(sd, ins, target=target, device="cuda")
    del ref.z
    m = _model(sd)
    eng = m.engine()
    shapes = [p.shape for p in m._ordered_params()]
    dins = [t.cuda() for t in ins]
    seed = ref.seed.float().cuda()
    results = [_abi_call(eng, dins, seed, shapes, tile, p) for p in (0, 3 * 50 * 59, 7 * 50 * 59)]
    for grads, gin in results:
        for a, b in zip(gin, results[0][1]):
            assert torch.equal(a, b)
        _check("pass size", ref, dict(zip(PARAM_NAMES, grads)), gin)


# ------------------------------------------------------------------ beyond the untiled limit
def test_12_mpx_image_beyond_the_untiled_limit():
    """1 x 3000 x 4000: the untiled training call refuses it; the windowed one runs it in bounded memory, and its
    gradients agree with float64 references computed on crops of radius 2 * RADIUS around sparse probes."""
    from waternet_b200 import WaterNetLibraryError
    from waternet_b200.engine import TRAIN_PASS_PIXELS
    n, h, w, tile = 1, 3000, 4000, 998
    sd = smooth_state_dict(71)
    ins = [t.cuda() for t in _images((n, h, w), 71)]
    with pytest.raises(WaterNetLibraryError):
        _model(sd)(*[t.clone().requires_grad_(True) for t in ins])
    rng = np.random.default_rng(71)
    from waternet_b200.engine import tile_geometry
    g = tile_geometry(h, w, tile, tile)
    cand = [(0, 0), (h - 1, w - 1), (0, w - 1), (h - 1, 0)]
    for y0, x0, (r0, r1), (c0, c1) in g["windows"]:
        cand += [(r0, c0), (r1 - 1, c1 - 1), (r0 - 1, c0), (y0, x0), (y0 + g["win_h"] - 1, x0 + g["win_w"] - 1)]
    cand += [(int(rng.integers(h)), int(rng.integers(w))) for _ in range(20)]
    probes = []
    for y, x in cand:
        if 0 <= y < h and 0 <= x < w and all(max(abs(y - a), abs(x - b)) > 4 * RADIUS + 1 for a, b in probes):
            probes.append((y, x))
    probes = probes[:24]
    signs = rng.choice([-1.0, 1.0], (len(probes), 3))
    grad = torch.zeros(n, 3, h, w, device="cuda")
    for (y, x), s in zip(probes, signs):
        grad[0, :, y, x] = torch.from_numpy(s).float().cuda()

    m = _model(sd, tile)
    leaves = [t.requires_grad_(True) for t in ins]
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = m(*leaves)
    out.backward(grad)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - held
    eng = m.engine()
    results = out.numel() * 4 + 4 * leaves[0].numel() * 4 + sum(p.numel() * 4 for p in m.parameters())
    budget = (eng.forward_tiled_workspace_bytes(n, h, w, tile, max_pass_pixels=TRAIN_PASS_PIXELS)
              + eng.backward_tiled_workspace_bytes(n, h, w, tile) + (1 << 30))
    print(f"\npeak beyond inputs {peak / 2**30:.2f} GiB, results {results / 2**30:.2f} GiB, "
          f"budget {budget / 2**30:.2f} GiB; untiled activations {eng.lib.wn_train_workspace_bytes(n, h, w) / 1e9:.0f} GB")
    assert peak - results <= budget

    params = {k: p.grad for k, p in m.named_parameters()}
    inputs = [t.grad for t in leaves]
    keep = torch.zeros(n, 1, h, w, dtype=torch.bool, device="cuda")
    sums = {k: 0 for k in PARAM_NAMES}
    msums = {k: 0 for k in PARAM_NAMES}
    crop = 2 * RADIUS
    for (y, x), s in zip(probes, signs):
        ya, yb, xa, xb = max(0, y - crop), min(h, y + crop + 1), max(0, x - crop), min(w, x + crop + 1)
        cg = torch.zeros(n, 3, yb - ya, xb - xa)
        cg[0, :, y - ya, x - xa] = torch.from_numpy(s).float()
        ref = reference(sd, [t.detach()[:, :, ya:yb, xa:xb] for t in ins], grad=cg, device="cuda")
        assert_relus_cannot_flip(ref.z)
        for k in PARAM_NAMES:
            sums[k] = sums[k] + ref.grads[k]
            msums[k] = msums[k] + ref.M[k]
        for name, gi, r, mm in zip(INPUT_NAMES, inputs, ref.input_grads, ref.M_inputs):
            assert_grad_close(gi[:, :, ya:yb, xa:xb], r, mm, TAU, f"12 Mpx probe ({y}, {x}) {name}")
        keep[:, :, max(0, y - RADIUS):y + RADIUS + 1, max(0, x - RADIUS):x + RADIUS + 1] = True
    for name, gi in zip(INPUT_NAMES, inputs):
        assert (gi.masked_select(~keep.expand_as(gi)) == 0).all(), name
    for k in PARAM_NAMES:
        assert_grad_close(params[k], sums[k], msums[k], TAU, f"12 Mpx {k}")
    print(f"12 Mpx: {len(probes)} probes")


# ------------------------------------------------------------------ autograd plumbing
def test_autograd_plumbing():
    n, h, w, tile = 1, 40, 60, 16
    sd = gated_state_dict(73)
    ins = [t.cuda() for t in _images((n, h, w), 73)]
    grad = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(74)).cuda()
    base = _native(sd, [t.cpu() for t in ins], grad.cpu(), grad_tile=tile)

    m = _model(sd, tile)  # inputs only: the parameters do not require grad and get None
    for p in m.parameters():
        p.requires_grad_(False)
    leaves = [t.clone().requires_grad_(True) for t in ins]
    m(*leaves).backward(grad)
    assert all(p.grad is None for p in m.parameters())
    for a, b in zip(leaves, base[2]):
        assert torch.equal(a.grad, b)

    m = _model(sd, tile)  # parameters only
    out = m(*ins)
    assert out.grad_fn is not None
    out.backward(grad)
    for k, p in m.named_parameters():
        assert torch.equal(p.grad, base[1][k]), k

    m = _model(sd, tile)  # some parameters frozen
    m.cmg.conv3.weight.requires_grad_(False)
    m(*ins).backward(grad)
    assert m.cmg.conv3.weight.grad is None and torch.equal(m.cmg.conv4.weight.grad, base[1]["cmg.conv4.weight"])

    m = _model(sd, tile)  # an input edited in place between forward and backward
    leaf = ins[0].clone().requires_grad_(True)
    x = leaf * 1.0
    out = m(x, *ins[1:])
    x.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.backward(grad)

    m = _model(sd, tile)  # parameters modified between forward and backward
    out = m(*ins)
    with torch.no_grad():
        m.cmg.conv1.weight.mul_(1.5)
    m(*[t[:, :, :8, :8] for t in ins]).sum()  # repacks the changed weights
    with pytest.raises(RuntimeError, match="modified between forward and backward"):
        out.backward(grad)
