"""The single-pass bf16 training arithmetic (WN_MODE_BF16) on the H100.

* Per launch, float64: through ``wn_debug_backward_layer`` with the handle in that mode, every training-forward
  activation, both seeds, the 11 data-gradient outputs, the parameter gradients and the input-gradient fold, each
  against the bf16 replay (bf16_replay) on the GPU's own decoded inputs and ReLU' decisions, within the replay bars and
  the exact-arithmetic bars.  Every plane buffer must be exactly bf16 (lo = 0): exactly one hi x hi product is taken.
* The relations of the entry points hold in this mode: windowed gradients equal untiled ones up to the order of the
  fp32 sums, ragged image i equals image i alone bit for bit, ragged windowed input gradients do not depend on
  max_pass_pixels.
* The default mode does not move: a handle set to WN_MODE_BF16 and back gives the bits of a fresh handle.
* Buffer bounds of the training rows in this mode; the setter; a short convergence run.
"""
import gc
import os

import pytest
import torch

import backward_reference as br
import bf16_replay as rp
import buffer_bounds as bb
import forward_reference as fr
from grad_reference import PARAM_NAMES
from test_backward_layers_gpu import _seed, _shapes, _stack_inputs, _train_forward
from test_buffer_bounds_gpu import _ok, _outputs, _run

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1, 1), (1, 19, 40), (2, 37, 53), (1, 300, 500), (300, 5, 7)]
FWD_BUFFER = {0: "a1", 1: "a2", 2: "a3", 3: "a4", 4: "a5", 5: "a6", 6: "a7", 7: "cm", 8: "r1", 9: "r2", 10: "refined"}
STACK_CASES = [("all", 0), ("cmg", 0), ("refiner", 0), ("refiner", 1), ("refiner", 2)]


def _mode():
    from waternet_b200 import _lib
    return _lib.MODE_BF16


@pytest.fixture(autouse=True)
def _free_device_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _report(name, value):
    path = os.environ.get("WN_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(f"{name} {value:.3e}\n")


def _engine(sd):
    from waternet_b200.engine import new_engine
    eng = new_engine("cuda:0")
    eng.pack_weights([sd[k].cuda() for k in PARAM_NAMES])
    return eng


def _read(eng, stack, which, ws, shape, grad):
    params = {k: torch.full(s, float("nan"), device="cuda") for k, s in _shapes().items()}
    own = {p for prefix in br.stack_params(stack, which) for p in (prefix + ".weight", prefix + ".bias")}
    grads = [params[k] if k in own else None for k in PARAM_NAMES]
    bufs = {}
    for name in br.stack_buffers(stack):
        b = br.NUMBER[name]
        bufs[name] = eng.debug_backward_layer(ws, shape, b, br.STACKS[stack], which, grad=grad if b >= 12 else None,
                                              grads=grads if b >= 14 else None, train_mode=_mode())
    return bufs, {k: params[k] for k in own}


WORST = {}


def _record(key, G, ref, tau, name, planes=False, exact_ref=None):
    rp.check(G, ref, tau, name, planes=planes)
    WORST[key] = max(WORST.get(key, (0.0, tau))[0], rp.excess(G, ref)), tau
    if exact_ref is not None:
        rp.check(G, exact_ref, rp.exact_bar(tau), name + " (exact)")


@pytest.mark.parametrize("stack,which", STACK_CASES)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_every_launch_against_the_bf16_replay(stack, which, shape):
    k = SHAPES.index(shape)
    weights = fr.WEIGHT_SETS[(k + STACK_CASES.index((stack, which))) % 4]
    kind = fr.INPUT_KINDS[k % 4]
    sd = fr.weight_set(weights)
    eng = _engine(sd)
    n, h, w = shape
    ins = _stack_inputs(stack, [t.cuda() for t in fr.make_inputs(kind, n, h, w, seed=k)], which)
    eng.set_train_mode(_mode())
    out, ws = _train_forward(eng, stack, which, ins)
    grad, _ = _seed("mse", out, k)
    bufs, params = _read(eng, stack, which, ws, shape, grad)
    label = f"{stack}/{which} {weights}/{kind} {shape}"
    sdc = {key: v.cuda() for key, v in sd.items()}
    rp.check(bufs["act0"], rp.types.SimpleNamespace(R=_bf16_cu(bufs["act0"]), M=bufs["act0"].double().abs(), F=0),
             2.0 ** -30, f"{label} act0", planes=True)
    for layer, name in FWD_BUFFER.items():
        if name not in bufs:
            continue
        src = bufs["act0"] if layer in (0, 8) else bufs[FWD_BUFFER[fr.INPUT_LAYER[layer]]]
        tau = rp.launch_tau(layer)
        _record(f"forward {name}", bufs[name], rp.layer_replay(sdc, layer, src), tau, f"{label} {name}",
                planes=name not in ("cm", "refined"), exact_ref=rp.layer_replay(sdc, layer, src, rounded=False))
    for name, ref in rp.seed_replay(stack, grad, bufs.get("cm"), bufs.get("refined"), which).items():
        _record(f"seed {name}", bufs[name], ref, rp.SEED_TAU, f"{label} {name}", planes=True)
    for li in br.DGRAD:
        if li in bufs:
            mask = br.DGRAD_MASK[li]
            g, m = bufs[br.DGRAD_INPUT[li]], bufs[mask] if mask else None
            _record(f"dgrad {li}", bufs[li], rp.dgrad_replay(sdc, li, g, m), rp.launch_tau(li), f"{label} {li}",
                    planes=True, exact_ref=rp.dgrad_replay(sdc, li, g, m, rounded=False))
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    for prefix in br.stack_params(stack, which):
        wref, bref = br.param_reference(prefix, bufs)
        li = br.WGRAD_SPECS[prefix][0]
        tau = rp.wgrad_tau(br.wgrad_pixels(li, n, h, w, sm))
        _record(f"wgrad {li}", params[prefix + ".weight"], wref, tau, f"{label} {prefix}.weight")
        _record("bias", params[prefix + ".bias"], bref, br.TAU["bias"], f"{label} {prefix}.bias")
    # the library's own backward in this mode writes the same parameter gradients; its input gradients are the fold
    saved = [(0, n, ws)]
    if stack == "all":
        grads, gin = eng.backward(grad, saved, list(_shapes().values()), want_input_grads=True, train_mode=_mode())
        real = dict(zip(PARAM_NAMES, grads))
    else:
        names = [key for key in PARAM_NAMES if key.rsplit(".", 1)[0] in set(br.stack_params(stack, which))]
        shp = [_shapes()[key] for key in names]
        if stack == "cmg":
            grads, gin = eng.confidence_maps_backward(grad, saved, shp, (True,) * 4, train_mode=_mode())
        else:
            grads, gin = eng.refine_backward(which, grad, saved, shp, (True, True), train_mode=_mode())
        real = dict(zip(names, grads))
    for key, t in params.items():
        assert torch.equal(t, real[key]), f"{label} {key}: debug call and backward differ"
    for t, (g, ref) in enumerate(zip(gin, br.fold_reference(stack, bufs.get("kD1"), bufs.get("kDR1"), which))):
        if stack == "all":
            _record("fold", g, ref, br.TAU["fold"], f"{label} input {t}")
        else:
            assert torch.equal(g, ref.R.float()), f"{label} input {t}"


def _bf16_cu(t):
    return t.double().float().bfloat16().double()


def test_zz_report_worst_replay_errors():
    """Prints the worst measured (|G - R| - F) / M per launch kind beside its bar (runs after the cases above)."""
    if not WORST:
        pytest.skip("no replay case ran in this session")
    for key, (v, tau) in sorted(WORST.items()):
        print(f"replay {key}: worst {v:.3e}  bar {tau:.3e}")
        _report(f"bf16 replay {key}", v)


# -------------------------------------------------------------------- the default mode does not move
def _grads_of(eng, ins, grad, tile=None, **kw):
    shapes = list(_shapes().values())
    if tile is None:
        out, saved = eng.forward_train(*ins, **kw)
        grads, gin = eng.backward(grad, saved, shapes, want_input_grads=True, **kw)
        return [out] + grads + gin
    grads, gin = eng.backward_tiled(grad, ins, shapes, tile, want_input_grads=True, max_pass_pixels=1 << 14, **kw)
    return grads + gin


def _submodule_grads(eng, ins, grad, **kw):
    names = [k for k in PARAM_NAMES if k.startswith("cmg.")]
    shp = [_shapes()[k] for k in names]
    maps, saved = eng.confidence_maps_train(*ins, **kw)
    g1, i1 = eng.confidence_maps_backward(grad, saved, shp, (True,) * 4, **kw)
    names = [k for k in PARAM_NAMES if k.startswith("ce_refiner.")]
    shp = [_shapes()[k] for k in names]
    out, saved = eng.refine_train(1, ins[0], ins[2], **kw)
    g2, i2 = eng.refine_backward(1, grad, saved, shp, (True, True), **kw)
    return [maps, out] + g1 + i1 + g2 + i2


def _ragged_grads(eng, items, grads_out, **kw):
    outs, saved = eng.forward_train_ragged(items, **kw)
    grads, gin = eng.backward_ragged(grads_out, saved, list(_shapes().values()), [(True,) * 4] * len(items), **kw)
    return outs + grads + [t for row in gin for t in row]


def _all_paths(eng, **kw):
    torch.manual_seed(1)
    ins = [torch.rand(2, 3, 37, 53, device="cuda") for _ in range(4)]
    grad = torch.randn(2, 3, 37, 53, device="cuda")
    items = [[torch.rand(1, 3, h, w, device="cuda") for _ in range(4)] for h, w in ((23, 17), (40, 31))]
    gouts = [torch.randn(1, 3, h, w, device="cuda") for h, w in ((23, 17), (40, 31))]
    return (_grads_of(eng, ins, grad, **kw) + _grads_of(eng, ins, grad, tile=(23, 29), **kw) +
            _submodule_grads(eng, ins, grad, **kw) + _ragged_grads(eng, items, gouts, **kw))


def test_default_mode_is_unchanged_by_a_round_trip_through_bf16():
    sd = fr.weight_set("default")
    fresh = _all_paths(_engine(sd))
    eng = _engine(sd)
    eng.set_train_mode(_mode())
    bf16 = _all_paths(eng, train_mode=_mode())
    eng.set_train_mode(1)
    again = _all_paths(eng)
    for k, (a, b) in enumerate(zip(fresh, again)):
        assert torch.equal(a, b), f"tensor {k} moved after a round trip through WN_MODE_BF16"
    assert any(not torch.equal(a, b) for a, b in zip(fresh, bf16)), "WN_MODE_BF16 computed the bf16x3 bits"


# -------------------------------------------------------------------- entry-point relations in this mode
def test_windowed_equals_untiled_up_to_bf16_rounding():
    """In bf16x3 the windowed gradients equal the untiled ones up to the order of the fp32 sums.  In single-pass bf16
    every window rounds its own share of a halo pixel's gradient planes to bf16 before the weight-gradient GEMM sums
    them, where the untiled pass rounds their sum once (the input gradients: the fold adds each window's bf16 share).
    So the results agree to a bf16 rounding, not to the last bits: the difference is within 2^-8 (the unit roundoff of
    one bf16 rounding) of each tensor in the 2-norm, and within 2^-6 of its largest element anywhere."""
    sd = fr.weight_set("trained")
    eng = _engine(sd)
    torch.manual_seed(2)
    ins = [torch.rand(2, 3, 61, 47, device="cuda") for _ in range(4)]
    grad = torch.randn(2, 3, 61, 47, device="cuda")
    untiled = _grads_of(eng, ins, grad, train_mode=_mode())[1:]
    tiled = _grads_of(eng, ins, grad, tile=(23, 29), train_mode=_mode())
    for name, a, b in zip(PARAM_NAMES + ["x", "wb", "he", "gc"], untiled, tiled):
        assert (a - b).norm().item() <= 2.0 ** -8 * a.norm().item(), name
        assert (a - b).abs().max().item() <= 2.0 ** -6 * a.abs().max().item(), name


def test_ragged_image_equals_image_alone_bit_for_bit():
    sd = fr.weight_set("stress")
    eng = _engine(sd)
    torch.manual_seed(3)
    sizes = ((23, 17), (40, 31), (5, 7))
    items = [[torch.rand(1, 3, h, w, device="cuda") for _ in range(4)] for h, w in sizes]
    gouts = [torch.randn(1, 3, h, w, device="cuda") for h, w in sizes]
    outs, saved = eng.forward_train_ragged(items, train_mode=_mode())
    _, gin = eng.backward_ragged(gouts, saved, list(_shapes().values()), [(True,) * 4] * 3, train_mode=_mode())
    for i, (it, g) in enumerate(zip(items, gouts)):
        out, sv = eng.forward_train(*it, train_mode=_mode())
        _, gi = eng.backward(g, sv, list(_shapes().values()), want_input_grads=True, train_mode=_mode())
        assert torch.equal(out, outs[i]), f"image {i} output"
        for t in range(4):
            assert torch.equal(gi[t], gin[i][t]), f"image {i} input gradient {t}"


def test_ragged_windowed_input_grads_do_not_depend_on_the_pass_size():
    sd = fr.weight_set("default")
    eng = _engine(sd)
    torch.manual_seed(4)
    sizes = ((61, 47), (37, 90))
    items = [[torch.rand(1, 3, h, w, device="cuda") for _ in range(4)] for h, w in sizes]
    gouts = [torch.randn(1, 3, h, w, device="cuda") for h, w in sizes]
    res = []
    for mpp in (1 << 12, 1 << 16):
        _, gin = eng.backward_ragged_tiled(gouts, items, list(_shapes().values()), (23, 29), [(True,) * 4] * 2,
                                           max_pass_pixels=mpp, train_mode=_mode())
        res.append(gin)
    for a, b in zip(res[0], res[1]):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


# -------------------------------------------------------------------- buffer bounds in this mode
BOUNDS_ROWS = ("train", "train_ragged", "confidence_maps_train", "refine_train", "backward_tiled",
               "confidence_maps_backward_tiled", "refine_backward_tiled", "backward_ragged_tiled")
BOUNDS = [(r, s) for r in bb.ROWS if r.name in BOUNDS_ROWS for s in r.specs if s.get("shape") != bb.BIG and
          not any(h * w > 1 << 20 for h, w in s.get("sizes", []))]


@pytest.fixture(scope="module")
def bounds_eng():
    from waternet_b200.engine import new_engine
    e = new_engine("cuda:0")
    e.pack_weights(bb.waternet_params())
    yield e


def test_bounds_rows_are_present():
    assert {r.name for r, _ in BOUNDS} == set(BOUNDS_ROWS)


@pytest.mark.parametrize("row,spec", BOUNDS, ids=[f"{r.name}-{bb.spec_id(s)}" for r, s in BOUNDS])
def test_training_rows_stay_inside_their_buffers(bounds_eng, row, spec):
    """Guards, the exact workspace at two offsets with different poison (the same bits, no NaN), one byte short
    refused, with the handle in WN_MODE_BF16."""
    eng = bounds_eng
    eng.set_train_mode(_mode())
    plan = row.build(spec)
    results = []
    for k, off in enumerate((0, 768)):
        rc, P, ws = _run(eng, row, spec, plan, offset=off, poison=k, ws_fill=k)
        _ok(eng, rc, P, ws, f"offset {off}")
        results.append(_outputs(plan, P))
        del P, ws
    for name, t in results[0].items():
        assert torch.equal(t.contiguous().view(-1).view(torch.uint8), results[1][name].contiguous().view(-1).view(
            torch.uint8)), name
        if t.dtype == torch.float32:
            assert not bool(torch.isnan(t).any()), name
    if row.ws:
        need = bb.workspace_bytes(eng.lib, row, spec)
        rc, P, ws = _run(eng, row, spec, plan, ws_bytes=need - 1)
        assert rc == -4, f"one byte short: code {rc}"


# -------------------------------------------------------------------- the setter
def test_setter_and_inference_modes():
    from waternet_b200 import _lib
    eng = _engine(fr.weight_set("default"))
    for bad in (-1, 0, 2, 4, 99):
        assert eng.lib.wn_set_train_mode(eng.handle, bad) == -1
        assert str(bad) in eng.lib.wn_last_error().decode()
    eng.set_train_mode(_lib.MODE_BF16)
    x = [torch.rand(1, 3, 16, 16, device="cuda") for _ in range(4)]
    with pytest.raises(_lib.WaterNetLibraryError):
        eng.forward(*x, mode=_lib.MODE_BF16)
    eng.set_train_mode(_lib.MODE_BF16X3)


def test_a_module_keeps_its_mode_across_another_modules_step():
    """A model's stacks share its engine's handle.  The refiner's bf16 step stays bf16 when the cmg takes a bf16x3
    step on the same handle between its forward and its backward: the mode travels in the autograd ctx."""
    from waternet_b200.net import WaterNet
    torch.manual_seed(5)
    ins = [torch.rand(1, 3, 33, 29, device="cuda") for _ in range(4)]
    m = WaterNet(train_precision="bf16")
    m.load_state_dict(fr.weight_set("default"))
    m = m.cuda().train()
    m.ce_refiner(ins[0], ins[2]).square().sum().backward()
    want = [p.grad.clone() for p in m.ce_refiner.parameters()]
    m.zero_grad()
    out = m.ce_refiner(ins[0], ins[2])
    m.train_precision = "bf16x3"
    m.cmg(*ins)[0].sum().backward()
    out.square().sum().backward()
    for p, w in zip(m.ce_refiner.parameters(), want):
        assert torch.equal(p.grad, w)
    # and the whole network: a bf16x3 step of the cmg between a bf16 forward and its backward
    m.train_precision = "bf16"
    m.zero_grad()
    m(*ins).square().sum().backward()
    want = [p.grad.clone() for p in m.parameters()]
    m.zero_grad()
    out = m(*ins)
    m.train_precision = "bf16x3"
    m.cmg(*ins)[1].sum().backward()
    m.zero_grad()
    out.square().sum().backward()
    for p, w in zip(m.parameters(), want):
        assert torch.equal(p.grad, w)


# -------------------------------------------------------------------- convergence
def test_short_synthetic_run_converges_like_bf16x3():
    from waternet_b200.net import WaterNet
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(0)
    n, h, w = 16, 112, 112
    data = [[torch.rand(n, 3, h, w, generator=g) for _ in range(4)] for _ in range(4)]
    target = [d[1] * 0.5 + d[2] * 0.3 + d[3] * 0.2 for d in data]
    curves = {}
    for tp in ("bf16x3", "bf16"):
        torch.manual_seed(0)
        m = WaterNet(train_precision=tp).cuda().train()
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        losses = []
        for epoch in range(3):
            tot = 0.0
            for d, t in zip(data, target):
                ins = [x.cuda() for x in d]
                loss = torch.nn.functional.mse_loss(m(*ins), t.cuda())
                opt.zero_grad()
                loss.backward()
                opt.step()
                tot += loss.item()
            losses.append(tot / len(data))
        curves[tp] = losses
    print("convergence", curves)
    for tp, c in curves.items():
        assert c[-1] < c[0], f"{tp}: the loss does not fall: {c}"
    for a, b in zip(curves["bf16x3"], curves["bf16"]):
        assert abs(a - b) <= 0.05 * a, curves
