"""Every launch of the training backward, element by element against float64 on the launch's own input.

Each case runs one training forward on the library, then reads back through ``wn_debug_backward_layer`` the saved
activations, the seeds and the output of every data-gradient launch, with the parameter gradients the backward wrote.
Each is checked with ``backward_reference``, |G - R| <= tau M, R and M computed in float64 on the device from the
decoded buffers the launch consumed.  The ReLU' masks are the GPU's own saved activations, so any weights can be used:
the stress, default, trained and graded sets, whose ReLUs do flip against a float64 forward and which the whole-network
checks of test_backward_gpu.py cannot use.  Shapes: 1 x 1, widths of 8 (mod 16), every height (mod 16), 2 x 37 x 53,
1 x 300 x 500, and the weight-gradient shapes 4 x 97 x 131, 1 x 385 x 577 (hundreds of tiles per CTA) and 300 x 5 x 7
(tiles that span images).  Seeds: an MSE seed against a random target, and sparse probes, whose every launch must be
exactly 0.0 outside the probes' receptive fields.  Stacks: the whole network, the cmg alone and each refiner alone.
"""
import ctypes
import gc
import os

import pytest
import torch

import backward_reference as br
import forward_reference as fr
from grad_reference import PARAM_NAMES, assert_grad_close
from test_backward_gpu import DENSE_SHAPES, PROBE_SHAPES, _probes
from test_forward_layers_gpu import EDGE_SHAPES

pytestmark = pytest.mark.gpu

SHAPES = EDGE_SHAPES + [s for s in DENSE_SHAPES if s in ((4, 97, 131), (1, 385, 577), (300, 5, 7))]
# the radius of each buffer's support around a pixel where the seed is nonzero: the sum of the kernel radii from the
# output back to that buffer (cmg conv8 .. conv1: 1, 1, 2, 3, 0, 1, 2, 3; refiners conv3 .. conv1: 1, 2, 3)
RADIUS = {"g8": 0, "gr3": 0, "kD8": 1, "kD7": 2, "kD6": 4, "kD5": 7, "kD4": 7, "kD3": 8, "kD2": 10, "kD1": 13,
          "kDR3": 1, "kDR2": 3, "kDR1": 6}


@pytest.fixture(autouse=True)
def _free_device_memory():
    torch.cuda.reset_peak_memory_stats()
    yield
    gc.collect()
    torch.cuda.empty_cache()
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def _report(name, value):
    """With WN_REPORT set to a file name: append the measured value (how the bars were set)."""
    path = os.environ.get("WN_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(f"{name} {value:.3e}\n")


def _model(sd):
    from waternet_b200.net import WaterNet
    m = WaterNet()
    m.load_state_dict(sd, strict=True)
    return m.cuda().train()


def _stack_inputs(stack, ins, which):
    return list(ins) if stack != "refiner" else [ins[0], ins[1 + which]]


def _train_forward(eng, stack, which, ins, fill=None):
    """One training forward call of the stack on the library: (out, workspace).  fill: byte value the workspace
    holds before the call (None: uninitialised)."""
    ins = eng._check_inputs(ins)
    n, _, h, w = ins[0].shape
    lib = eng.lib
    nbytes = lib.wn_train_workspace_bytes(n, h, w) if stack == "all" else \
        lib.wn_submodule_train_workspace_bytes(n, h, w, br.STACKS[stack])
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda") if fill is None else \
        torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda")
    out = torch.empty(n, 3, h, w, device="cuda")
    st = (ctypes.c_int64 * (4 * len(ins)))(*[s for t in ins for s in t.stride()])
    p = [t.data_ptr() for t in ins]
    stream = torch.cuda.current_stream().cuda_stream
    if stack == "all":
        rc = lib.wn_forward_train(eng.handle, *p, st, out.data_ptr(), n, h, w, ws.data_ptr(), ws.numel(), stream)
    elif stack == "cmg":
        rc = lib.wn_confidence_maps_train(eng.handle, *p, st, out.data_ptr(), n, h, w, ws.data_ptr(), ws.numel(),
                                          stream)
    else:
        rc = lib.wn_refine_train(eng.handle, which, *p, st, out.data_ptr(), n, h, w, ws.data_ptr(), ws.numel(), stream)
    from waternet_b200 import _lib
    _lib.check(rc, f"training forward of {stack}")
    return out, ws


def _seed(kind, out, seed):
    n, _, h, w = out.shape
    if kind == "mse":
        target = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(seed)).cuda()
        return 2 * (out - target) / out.numel(), None
    probes = _probes(n, h, w, h * w + seed)
    grad = torch.zeros(n, 3, h, w)
    gen = torch.Generator().manual_seed(seed)
    for i, y, x in probes:
        grad[i, :, y, x] = torch.randint(0, 2, (3,), generator=gen).float() * 2 - 1
    return grad.cuda(), probes


def _read(eng, stack, which, ws, shape, grad):
    """Every buffer of the stack's training pass and the parameter gradients of its last launch's call."""
    params = {k: torch.full(s, float("nan"), device="cuda") for k, s in _shapes().items()}
    own = {p for prefix in br.stack_params(stack, which) for p in (prefix + ".weight", prefix + ".bias")}
    grads = [params[k] if k in own else None for k in PARAM_NAMES]
    bufs = {}
    for name in br.stack_buffers(stack):
        b = br.NUMBER[name]
        bufs[name] = eng.debug_backward_layer(ws, shape, b, br.STACKS[stack], which,
                                              grad=grad if b >= 12 else None, grads=grads if b >= 14 else None)
    return bufs, {k: params[k] for k in own}


def _shapes():
    from oracle import forward as ofw
    return dict(ofw.state_dict_spec())


def _real_backward(eng, stack, which, ws, shape, grad):
    """The library's own backward on the same workspace (wn_backward or the sub-module's): (params, input grads)."""
    n = shape[0]
    saved = [(0, n, ws)]
    if stack == "all":
        grads, gin = eng.backward(grad, saved, [s for _, s in _shapes().items()], want_input_grads=True)
        return dict(zip(PARAM_NAMES, grads)), gin
    prefixes = set(br.stack_params(stack, which))
    names = [k for k in PARAM_NAMES if k.rsplit(".", 1)[0] in prefixes]  # state-dict order, as the library writes
    shapes = [_shapes()[k] for k in names]
    if stack == "cmg":
        grads, gin = eng.confidence_maps_backward(grad, saved, shapes, (True,) * 4)
    else:
        grads, gin = eng.refine_backward(which, grad, saved, shapes, (True, True))
    return dict(zip(names, grads)), gin


def _check_case(eng, sd, stack, ins, seed_kind, worst, label, which=0, fill=None, seed=0):
    """Every seed, launch, parameter gradient and input gradient of one backward; worst[key] keeps the largest
    |G - R| / M (for the weight gradients: over wgrad_tau(P), and the P it was measured at)."""
    cu = _stack_inputs(stack, [t.cuda() for t in ins], which)
    n, _, h, w = cu[0].shape
    shape = (n, h, w)
    out, ws = _train_forward(eng, stack, which, cu, fill)
    grad, probes = _seed(seed_kind, out, seed)
    bufs, params = _read(eng, stack, which, ws, shape, grad)
    for name, t in bufs.items():
        assert t.shape == (n, br.CHANNELS[name], h, w) and torch.isfinite(t).all(), (label, name)

    def record(key, ref, G, tau, name):
        assert_grad_close(G.double(), ref.R, ref.M, tau, f"{label} {name}")
        worst[key] = max(worst.get(key, 0.0), br.ratio(G, ref) * (br.wgrad_tau(0) / tau if "wgrad" in key else 1))

    for name, ref in br.seed_reference(stack, grad, bufs.get("cm"), bufs.get("refined"), which).items():
        record(f"seed {name}", ref, bufs[name], br.TAU["seed"], name)
    for li in br.DGRAD:
        if li in bufs:
            mask = br.DGRAD_MASK[li]
            ref = br.dgrad_reference(sd, li, bufs[br.DGRAD_INPUT[li]], bufs[mask] if mask else None)
            record(f"dgrad {li}", ref, bufs[li], br.TAU["dgrad"], li)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    for prefix in br.stack_params(stack, which):
        wref, bref = br.param_reference(prefix, bufs)
        li = br.WGRAD_SPECS[prefix][0]
        pix = br.wgrad_pixels(li, n, h, w, sm)
        record(f"wgrad {li}", wref, params[prefix + ".weight"], br.wgrad_tau(pix), prefix + ".weight")
        _report(f"wgrad_P {label} {prefix} P={pix}", br.ratio(params[prefix + ".weight"], wref))
        record("bias", bref, params[prefix + ".bias"], br.TAU["bias"], prefix + ".bias")
    # the parameter gradients the debug calls wrote are those of the library's backward, bit for bit; its input
    # gradients are the fold of the decoded first-layer launches
    real, gin = _real_backward(eng, stack, which, ws, shape, grad)
    for k, t in params.items():
        assert torch.equal(t, real[k]), f"{label} {k}: debug call and backward differ"
    folds = br.fold_reference(stack, bufs.get("kD1"), bufs.get("kDR1"), which)
    for t, (g, ref) in enumerate(zip(gin, folds)):
        if stack == "all":
            record("fold", ref, g, br.TAU["fold"], f"input {t}")
        else:  # extract_input_grads_kernel adds hi + lo of the one buffer as the decode does
            assert torch.equal(g, ref.R.float()), f"{label} input {t}"
    if probes is not None:
        keep = {}
        for name, r in RADIUS.items():
            if name not in bufs:
                continue
            if r not in keep:
                k = torch.zeros(n, 1, h, w, dtype=torch.bool)
                for i, y, x in probes:
                    k[i, :, max(0, y - r):y + r + 1, max(0, x - r):x + r + 1] = True
                keep[r] = k.cuda()
            leak = bufs[name].masked_select(~keep[r].expand_as(bufs[name]))
            assert (leak == 0).all(), f"{label} {name}: {(leak != 0).sum().item()} nonzero elements outside the probes' support"
    return bufs


def _print(title, worst):
    print(f"{title}: worst |G - R| / M (weight gradients: scaled to the bar at P = 0) " +
          " ".join(f"{k}={v:.2e}" for k, v in sorted(worst.items())))
    for k, v in worst.items():
        _report(f"{title} {k}", v)


def test_every_buffer_at_tile_edges():
    """Stress weights, random floats, the whole network with an MSE seed, at every shape of SHAPES."""
    sd = fr.weight_set("stress", 11)
    eng = _model(sd).engine()
    worst = {}
    for n, h, w in SHAPES:
        _check_case(eng, sd, "all", fr.make_inputs("floats", n, h, w, h * 1000 + w), "mse", worst, f"{(n, h, w)}",
                    seed=h + w)
    _print("shapes", worst)


@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
def test_every_buffer_per_weight_set_and_input(weights):
    """Each weight set with level, float, dark-float and dark-level inputs, the whole network at 2 x 37 x 53."""
    sd = fr.weight_set(weights, 2)
    eng = _model(sd).engine()
    worst = {}
    for i, kind in enumerate(fr.INPUT_KINDS):
        _check_case(eng, sd, "all", fr.make_inputs(kind, 2, 37, 53, 50 + i), "mse", worst, f"{weights} {kind}",
                    seed=i)
    _print(weights, worst)


@pytest.mark.parametrize("shape", PROBE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_probe_seeds_stay_in_their_support(shape):
    """Isolated +-1 seeds: every launch is exact 0.0 outside the probes' receptive fields and within its bar inside."""
    sd = fr.weight_set("trained", 4)
    eng = _model(sd).engine()
    worst = {}
    _check_case(eng, sd, "all", fr.make_inputs("floats", *shape, 5), "probes", worst, f"probes {shape}", seed=7)
    _print(f"probes {shape}", worst)


@pytest.mark.parametrize("stack,which", [("cmg", 0), ("refiner", 0), ("refiner", 1), ("refiner", 2)])
def test_submodule_stacks(stack, which):
    """The cmg alone (seed_kernel's maps seed) and each refiner alone (its refine seed: the other refiners'
    columns exactly 0), with MSE and probe seeds, on the stress and default weights."""
    worst = {}
    for weights in ("stress", "default"):
        sd = fr.weight_set(weights, 6)
        eng = _model(sd).engine()
        for kind, shape in (("mse", (2, 37, 53)), ("probes", (4, 97, 131))):
            bufs = _check_case(eng, sd, stack, fr.make_inputs("floats", *shape, 8), kind, worst,
                               f"{stack} {which} {weights} {kind}", which, seed=9)
            if stack == "refiner":
                others = [c for r in range(3) if r != which for c in range(3 * r, 3 * r + 3)]
                assert (bufs["gr3"][:, others] == 0).all() and (bufs["gr3"][:, 9:] == 0).all()
    _print(f"{stack} {which}", worst)


@pytest.mark.parametrize("stack,which", [("all", 0), ("cmg", 0), ("refiner", 1)])
def test_stale_workspace(stack, which):
    """A workspace of 0xFF bytes (NaN in bf16 and fp32) before the training forward: every buffer is written before
    it is read.  With 8-bit level inputs the first layers' weight gradients still read act0's lo planes (zeros)."""
    sd = fr.weight_set("default", 12)
    eng = _model(sd).engine()
    worst = {}
    for kind in ("levels", "floats"):
        bufs = _check_case(eng, sd, stack, fr.make_inputs(kind, 2, 37, 53, 13), "mse", worst, f"stale {stack} {kind}",
                           which, fill=0xFF, seed=14)
        if kind == "levels":
            assert torch.equal(bufs["act0"], bufs["act0"].round())
    _print(f"stale {stack}", worst)


def test_saved_activations_equal_the_debug_forward():
    """The training forward keeps, bit for bit, what wn_debug_forward_layer returns in bf16x3 for layers 0..10; act0
    holds the snapped v * 255 operands (exactly the levels for 8-bit inputs) and zeros in channels 12..15."""
    from waternet_b200 import _lib
    sd = fr.weight_set("trained", 15)
    eng = _model(sd).engine()
    names = ["a1", "a2", "a3", "a4", "a5", "a6", "a7", "cm", "r1", "r2", "refined"]
    for kind in ("floats", "levels"):
        cu = [t.cuda() for t in fr.make_inputs(kind, 2, 37, 53, 16)]
        _, ws = _train_forward(eng, "all", 0, cu)
        for layer, name in enumerate(names):
            saved = eng.debug_backward_layer(ws, (2, 37, 53), br.NUMBER[name])
            fwd = eng.debug_layer(*cu, layer=layer, mode=_lib.MODE_BF16X3)
            assert torch.equal(saved, fwd), (kind, name)
        act0 = eng.debug_backward_layer(ws, (2, 37, 53), br.NUMBER["act0"]).double()
        v = torch.cat(cu, 1).double() * 255
        assert (act0[:, 12:] == 0).all()
        if kind == "levels":
            assert torch.equal(act0[:, :12], v.round())
        else:
            assert ((act0[:, :12] - v).abs() <= 2.0 ** -15 * v.abs()).all()


@pytest.mark.parametrize("stack,which", [("all", 0), ("cmg", 0), ("refiner", 2)])
def test_debug_calls_equal_the_model_backward(stack, which):
    """The parameter gradients the debug calls write equal those of model(*ins) / out.backward(grad) bit for bit; the
    input gradients are the decoded first-layer launches (the sub-modules: bit for bit) or their fp32 fold."""
    sd = fr.weight_set("stress", 17)
    m = _model(sd)
    eng = m.engine()
    ins = [t.cuda() for t in fr.make_inputs("floats", 2, 37, 53, 18)]
    grad = torch.randn(2, 3, 37, 53, generator=torch.Generator().manual_seed(19)).cuda()
    leaves = [t.clone().requires_grad_(True) for t in _stack_inputs(stack, ins, which)]
    if stack == "all":
        m(*leaves).backward(grad)
    elif stack == "cmg":
        torch.autograd.backward(m.cmg(*leaves), [grad[:, r:r + 1] for r in range(3)])
    else:
        getattr(m, ["wb_refiner", "ce_refiner", "gc_refiner"][which])(*leaves).backward(grad)
    named = dict(m.named_parameters())
    _, ws = _train_forward(eng, stack, which, _stack_inputs(stack, ins, which))
    bufs, params = _read(eng, stack, which, ws, (2, 37, 53), grad)
    for k, t in params.items():
        assert torch.equal(t, named[k].grad), k
    for t, (leaf, ref) in enumerate(zip(leaves, br.fold_reference(stack, bufs.get("kD1"), bufs.get("kDR1"), which))):
        if stack == "all":
            assert_grad_close(leaf.grad.double(), ref.R, ref.M, br.TAU["fold"], f"input {t}")
        else:
            assert torch.equal(leaf.grad, ref.R.float()), t


def test_cpu_and_cuda_references_agree():
    """The float64 references do not depend on the device they run on."""
    sd = fr.weight_set("graded", 3)
    torch.manual_seed(0)
    bufs = {name: torch.rand(1, c, 13, 21) - (0.3 if name in br.DGRAD + ["g8", "gr3"] else 0.0)
            for name, c in br.CHANNELS.items()}
    grad = torch.randn(1, 3, 13, 21)

    def same(cpu, gpu, label):
        bar = cpu.M
        assert ((gpu.R.cpu() - cpu.R).abs() <= 1e-11 * bar).all(), label
        assert ((gpu.M.cpu() - cpu.M).abs() <= 1e-11 * bar).all(), label

    gbufs = {k: v.cuda() for k, v in bufs.items()}
    for stack in ("all", "cmg", "refiner"):
        cpu = br.seed_reference(stack, grad, bufs["cm"], bufs["refined"], 1)
        gpu = br.seed_reference(stack, grad.cuda(), gbufs["cm"], gbufs["refined"], 1)
        for k in cpu:
            same(cpu[k], gpu[k], k)
    for li in br.DGRAD:
        mask = br.DGRAD_MASK[li]
        same(br.dgrad_reference(sd, li, bufs[br.DGRAD_INPUT[li]], bufs[mask] if mask else None),
             br.dgrad_reference(sd, li, gbufs[br.DGRAD_INPUT[li]], gbufs[mask] if mask else None), li)
    for prefix in br.WGRAD_SPECS:
        for c, g in zip(br.param_reference(prefix, bufs), br.param_reference(prefix, gbufs)):
            same(c, g, prefix)
