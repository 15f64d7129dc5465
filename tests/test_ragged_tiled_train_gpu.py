"""The windowed recompute backward of a ragged batch on the GPU: WaterNet.forward_many under grad_tile
(wn_forward_ragged + wn_backward_ragged_tiled).  Outputs and input gradients must equal, bit for bit, what the
per-item windowed path (model(*item) under the same grad_tile) gives; a list of one size must equal wn_backward_tiled
of the stacked batch in every gradient; parameter gradients must match the float64 sum over the images.  Workspaces
are pre-filled with 0xFF (a bf16 NaN in every operand plane), so a slot pixel beyond a window that is not masked
shows."""
import gc

import pytest
import torch

import grad_reference as gr

pytestmark = pytest.mark.gpu

TILE = 20  # < 2 * 13: a pixel of a large image lies in three or more windows per axis


@pytest.fixture(autouse=True)
def _free_device_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _model(sd, grad_tile=TILE, precision="bf16x3"):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision, grad_tile=grad_tile)
    m.load_state_dict(sd, strict=True)
    return m.cuda().train()


def _rand(shape, g, levels):
    if levels:
        return torch.randint(0, 256, shape, generator=g).float() / 255
    return torch.rand(shape, generator=g)


def _mixed_items(seed):
    """1 x 1, widths of 8 (mod 16), odd sizes, an item of two images (one of levels, one not), a zero-pixel item,
    channels_last and strided inputs, level and non-level items, and images of many windows."""
    g = torch.Generator().manual_seed(seed)
    spec = [((1, 3, 1, 1), True), ((1, 3, 8, 24), False), ((1, 3, 37, 53), True), ((1, 3, 0, 5), False),
            ((1, 3, 150, 200), False), ((1, 3, 61, 45), True), ((1, 3, 97, 130), False)]
    items = [tuple(_rand(s, g, lv).cuda() for _ in range(4)) for s, lv in spec]
    pair = [torch.cat([_rand((1, 3, 45, 71), g, True), _rand((1, 3, 45, 71), g, False)], 0).cuda()
            for _ in range(4)]
    items.insert(3, tuple(pair))
    items[5] = tuple(t.contiguous(memory_format=torch.channels_last) for t in items[5])
    items[7] = tuple(torch.cat([t, t.flip(3)], 3)[..., 1::2] for t in items[7])  # strided views
    return items


def _poison(eng):
    eng._train_ragged_workspace = lambda n: torch.full((int(n),), 0xFF, dtype=torch.uint8, device=eng.device)


def _poison_forward(eng, sizes, tile, max_pass):
    from waternet_b200 import _lib
    nbytes = eng.forward_ragged_workspace_bytes(sizes, tile, _lib.MODE_BF16X3, max_pass)
    eng._ws["forward"] = torch.full((int(nbytes) + 4096,), 0xFF, dtype=torch.uint8, device=eng.device)


def _sizes(items):
    return [(t[0].shape[2], t[0].shape[3]) for t in items for _ in range(t[0].shape[0]) if t[0].shape[2] * t[0].shape[3]]


def _equal(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not torch.equal(a, b):
        d = (a != b).nonzero()
        raise AssertionError(f"{what}: {len(d)} elements differ, first at {tuple(d[0].tolist())}: "
                             f"{a[tuple(d[0])].item()!r} vs {b[tuple(d[0])].item()!r}")


def _grads_out(items, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(tuple(it[0].shape), generator=g).cuda() for it in items]


def _per_item(model, items, grads_out):
    """The path forward_many took before: model(*item) under grad_tile, one item at a time."""
    outs, gins, gpars = [], [], []
    for it, go in zip(items, grads_out):
        if it[0].numel() == 0:  # model(...) of an empty item records no graph
            outs.append(torch.empty_like(go))
            gins.append([torch.zeros_like(t) for t in it])
            gpars.append([torch.zeros_like(p) for p in model.parameters()])
            continue
        leaves = [t.detach().clone().requires_grad_(True) for t in it]
        model.zero_grad(set_to_none=True)
        out = model(*leaves)
        out.backward(go)
        outs.append(out.detach())
        gins.append([t.grad for t in leaves])
        gpars.append([p.grad.clone() for p in model.parameters()])
    torch.cuda.synchronize()
    model.zero_grad(set_to_none=True)
    return outs, gins, gpars


# ------------------------------------------------------------------ bits against the per-item windowed path
@pytest.mark.parametrize("max_pass", [None, 5000])
def test_outputs_and_input_gradients_equal_the_per_item_path(max_pass):
    """max_pass None: forward_many as a user calls it (TRAIN_PASS_PIXELS slot pixels per pass).  5000: the engine
    calls at a pass of two 46 x 46 windows, which cuts through the windows of every large image."""
    from waternet_b200 import _lib
    from waternet_b200.engine import TRAIN_PASS_PIXELS
    sd = gr.gated_state_dict(21)
    model = _model(sd)
    eng = model.engine()
    items = _mixed_items(5)
    grads_out = _grads_out(items, 6)
    sizes = _sizes(items)
    _poison(eng)
    _poison_forward(eng, sizes, TILE, max_pass or TRAIN_PASS_PIXELS)
    if max_pass is None:
        leaves = [tuple(t.detach().clone().requires_grad_(True) for t in it) for it in items]
        outs = model.forward_many(*[list(t) for t in zip(*leaves)])
        torch.autograd.backward(outs, grads_out)
        outs = [o.detach() for o in outs]
        gin = [[t.grad for t in it] for it in leaves]
    else:
        shapes = [p.shape for p in model.parameters()]
        outs = eng.forward_ragged(items, TILE, _lib.MODE_BF16X3, max_pass_pixels=max_pass)
        from waternet_b200.engine import ragged_plan
        assert len(ragged_plan(sizes, TILE, TILE, max_pass)) > 10
        _, gin = eng.backward_ragged_tiled(grads_out, items, shapes, TILE, [(True,) * 4] * len(items), max_pass)
    torch.cuda.synchronize()
    del eng._train_ragged_workspace
    a_out, a_gin, _ = _per_item(model, items, grads_out)
    for i in range(len(items)):
        _equal(outs[i], a_out[i], f"output of item {i} {tuple(items[i][0].shape)}")
        for t in range(4):
            _equal(gin[i][t], a_gin[i][t], f"d/d{gr.INPUT_NAMES[t]} of item {i} {tuple(items[i][0].shape)}")


def test_a_list_of_one_size_equals_the_windowed_backward_of_the_batch():
    """Equal sizes give backward_tiled's plan (the same windows, order and passes, slot = window), so every gradient,
    the parameters' included, equals wn_backward_tiled of the stacked batch bit for bit."""
    from waternet_b200.engine import ragged_plan
    sd = gr.smooth_state_dict(31)
    model = _model(sd)
    eng = model.engine()
    g = torch.Generator().manual_seed(32)
    n, h, w, tile, max_pass = 3, 90, 130, 40, 20_000
    batch = [torch.rand((n, 3, h, w), generator=g).cuda() for _ in range(4)]
    go = torch.randn((n, 3, h, w), generator=g).cuda()
    shapes = [p.shape for p in model.parameters()]
    assert len(ragged_plan([(h, w)] * n, tile, tile, max_pass)) == 6
    ref_par, ref_in = eng.backward_tiled(go, batch, shapes, tile, want_input_grads=True, max_pass_pixels=max_pass)
    _poison(eng)
    items = [tuple(t[i:i + 1] for t in batch) for i in range(n)]
    par, gin = eng.backward_ragged_tiled([go[i:i + 1] for i in range(n)], items, shapes, tile,
                                         [(True,) * 4] * n, max_pass)
    torch.cuda.synchronize()
    for k, name in enumerate(gr.PARAM_NAMES):
        _equal(par[k], ref_par[k], name)
    for i in range(n):
        for t in range(4):
            _equal(gin[i][t], ref_in[t][i:i + 1], f"d/d{gr.INPUT_NAMES[t]} of image {i}")


# ------------------------------------------------------------------ parameter gradients against float64
@pytest.mark.parametrize("sd_kind", ["smooth", "gated"])
def test_parameter_gradients_match_the_summed_fp64_references(sd_kind):
    sd = (gr.smooth_state_dict if sd_kind == "smooth" else gr.gated_state_dict)(41)
    model = _model(sd)
    g = torch.Generator().manual_seed(42)
    sizes = [(8, 24), (37, 53), (70, 90), (45, 16)]
    items = [tuple(_rand((1, 3, h, w), g, i % 2 == 0).cuda() for _ in range(4)) for i, (h, w) in enumerate(sizes)]
    grads_out = _grads_out(items, 43)
    _poison(model.engine())
    outs = model.forward_many(*[list(t) for t in zip(*items)])
    torch.autograd.backward(outs, grads_out)
    torch.cuda.synchronize()
    gpar = [p.grad.clone() for p in model.parameters()]
    del model.engine()._train_ragged_workspace
    _, _, a_gpar = _per_item(model, items, grads_out)
    refs = [gr.reference(sd, it, grad=go, device="cuda") for it, go in zip(items, grads_out)]
    for r in refs:
        gr.assert_relus_cannot_flip(r.z)
    worst = 0.0
    for k, name in enumerate(gr.PARAM_NAMES):
        R = sum(r.grads[name] for r in refs)
        M = sum(r.M[name] for r in refs)
        worst = max(worst, gr.assert_grad_close(gpar[k], R, M, gr.TAU, name))
        gr.assert_grad_close(gpar[k], sum(p[k].double() for p in a_gpar), M, gr.TAU, name + " (per-item sum)")
    print(f"worst |G - R| / M: {worst:.3g}")


# ------------------------------------------------------------------ autograd plumbing
def test_partial_requires_grad_routes_gradients():
    sd = gr.smooth_state_dict(51)
    model = _model(sd)
    items = _mixed_items(52)[:4]
    req = [(True, False, False, True), (False,) * 4, (False, True, False, False), (True,) * 4]
    leaves = [tuple(t.clone().requires_grad_(r) for t, r in zip(it, rq)) for it, rq in zip(items, req)]
    for p in model.wb_refiner.parameters():
        p.requires_grad_(False)
    outs = model.forward_many(*[list(t) for t in zip(*leaves)])
    sum((o * (k + 1)).square().sum() for k, o in enumerate(outs)).backward()
    assert all(p.grad is None for p in model.wb_refiner.parameters())
    assert all(p.grad is not None for p in model.cmg.parameters())
    for k in range(len(items)):
        lv = tuple(t.clone().requires_grad_(r) for t, r in zip(items[k], req[k]))
        ((model(*lv) * (k + 1)).square().sum()).backward()
        for t in range(4):
            if req[k][t]:
                _equal(leaves[k][t].grad, lv[t].grad, f"item {k} input {t}")
            else:
                assert leaves[k][t].grad is None


def test_parameters_modified_between_forward_and_backward_raise():
    model = _model(gr.smooth_state_dict(61))
    items = _mixed_items(62)[:3]
    outs = model.forward_many(*[list(t) for t in zip(*items)])
    with torch.no_grad():
        model.cmg.conv1.bias.add_(0.01)
    model.engine()  # repack the edited weights
    with pytest.raises(RuntimeError, match="modified between forward and backward"):
        sum(o.sum() for o in outs).backward()


def test_fp32_with_grad_tile_is_refused():
    model = _model(gr.smooth_state_dict(63))
    items = _mixed_items(64)[:2]
    model.precision = "fp32"
    with pytest.raises(ValueError, match="tensor cores"):
        model.forward_many(*[list(t) for t in zip(*items)])


def test_a_window_over_the_pass_limit_raises_at_the_forward_call():
    from waternet_b200 import WaterNetLibraryError
    model = _model(gr.smooth_state_dict(65), grad_tile=2900)
    items = [tuple(torch.rand(1, 3, 16, 16, device="cuda") for _ in range(4)),
             tuple(torch.rand(1, 3, 2900, 2900, device="cuda") for _ in range(4))]  # 8.41 M > 8 Mi pixels
    with pytest.raises(WaterNetLibraryError, match="grad_tile"):
        model.forward_many(*[list(t) for t in zip(*items)])


# ------------------------------------------------------------------ bounded memory
def test_a_12_mpx_image_among_small_ones_trains_in_bounded_memory():
    """One 3000 x 4000 image and 30 small ones: the untiled ragged step cannot hold them; the windowed one peaks
    within one pass of the forward and the backward beyond its inputs and results."""
    from waternet_b200 import _lib
    from waternet_b200.engine import TRAIN_PASS_PIXELS
    tile = 998
    model = _model(gr.smooth_state_dict(71), grad_tile=tile)
    g = torch.Generator().manual_seed(72)
    sizes = [(3000, 4000)] + [(32 + 7 * k, 200 - 5 * k) for k in range(30)]
    items = [tuple(torch.rand(1, 3, h, w, generator=g).cuda().requires_grad_(True) for _ in range(4))
             for h, w in sizes]
    eng = model.engine()
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    outs = model.forward_many(*[list(t) for t in zip(*items)])
    sum(o.sum() for o in outs).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - held
    px = sum(h * w for h, w in sizes)
    results = px * 3 * 4 * (1 + 4) + sum(p.numel() * 4 for p in model.parameters())
    budget = (eng.forward_ragged_workspace_bytes(sizes, tile, _lib.MODE_BF16X3, TRAIN_PASS_PIXELS)
              + eng.backward_ragged_tiled_workspace_bytes(sizes, tile) + (1 << 30))
    untiled = px * 5616  # kTrainBytesPerPixel: the activations the untiled step keeps, before slot padding
    print(f"\npeak beyond inputs {peak / 2**30:.2f} GiB, results {results / 2**30:.2f} GiB, budget "
          f"{budget / 2**30:.2f} GiB; the untiled activations alone {untiled / 1e9:.0f} GB")
    assert peak - results <= budget < untiled
    assert all(torch.isfinite(t.grad).all() for it in items for t in it)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


# ------------------------------------------------------------------ train.py
def test_train_py_native_size_with_grad_tile_writes_its_artefacts(tmp_path):
    import json
    import os
    import shutil
    import subprocess
    import sys

    from conftest import ROOT
    shutil.copy(os.path.join(ROOT, "train.py"), tmp_path / "train.py")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(ROOT), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, str(tmp_path / "train.py"), "--synthetic", "--native-size", "--grad-tile",
                          "48", "--epochs", "1", "--height", "64", "--width", "64", "--seed", "0"], cwd=tmp_path,
                         env=env, capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    run = tmp_path / "training" / "0"
    for name in ("last.pt", "metrics-train.csv", "metrics-val.csv", "config.json"):
        assert (run / name).is_file(), name
    config = json.loads((run / "config.json").read_text())
    assert config["native_size"] is True
    rows = (run / "metrics-train.csv").read_text().strip().splitlines()
    assert len(rows) == 2  # header + 1 epoch
