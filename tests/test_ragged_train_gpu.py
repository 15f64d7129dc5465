"""Ragged batches of fp32 tensors on the GPU: WaterNet.forward_many (wn_forward_ragged) and the ragged training step
(wn_forward_train_ragged / wn_backward_ragged).  Every image's output and input gradients must equal, bit for bit,
what the per-image calls give; the parameter gradients must match the float64 sum over the images.  Workspaces are
pre-filled with 0xFF (a bf16 NaN in every operand plane), so a slot pixel beyond an image that is not masked shows."""
import pytest
import torch

import grad_reference as gr
from oracle import forward as ofw

pytestmark = pytest.mark.gpu

# 1 x 1, widths of 8 (mod 16), odd sizes, an empty image; the slot is the per-axis maximum (113 x 117)
SIZES = [(1, 1), (8, 24), (37, 53), (113, 117), (0, 5), (24, 40), (64, 72), (5, 113)]


def _model(sd, precision="bf16x3"):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def _inputs(sizes, seed, levels):
    """Four (1,3,h,w) inputs per size: 8-bit levels (u/255) where levels(i), uniform floats elsewhere."""
    g = torch.Generator().manual_seed(seed)
    items = []
    for i, (h, w) in enumerate(sizes):
        if levels(i):
            ts = [torch.randint(0, 256, (1, 3, h, w), generator=g).float() / 255 for _ in range(4)]
        else:
            ts = [torch.rand((1, 3, h, w), generator=g) for _ in range(4)]
        items.append(tuple(t.cuda() for t in ts))
    return items


def _poison_forward_workspace(eng, nbytes):
    eng._ws["forward"] = torch.full((int(nbytes) + 4096,), 0xFF, dtype=torch.uint8, device=eng.device)


def _poison_train_workspaces(eng):
    eng._train_ragged_workspace = lambda n: torch.full((int(n),), 0xFF, dtype=torch.uint8, device=eng.device)


def _equal(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not torch.equal(a, b):
        d = (a != b).nonzero()
        raise AssertionError(f"{what}: {len(d)} elements differ, first at {tuple(d[0].tolist())}: "
                             f"{a[tuple(d[0])].item()!r} vs {b[tuple(d[0])].item()!r}")


@pytest.mark.parametrize("precision", ["default", "bf16x3"])
@pytest.mark.parametrize("levels", ["all", "none", "mixed"])
def test_forward_many_matches_model_per_image(precision, levels):
    model = _model(ofw.synthetic_state_dict(3, 3.0), precision).eval()
    sel = {"all": lambda i: True, "none": lambda i: False, "mixed": lambda i: i % 2 == 0}[levels]
    items = _inputs(SIZES, 11, sel)
    eng = model.engine()
    _poison_forward_workspace(eng, eng.forward_ragged_workspace_bytes([(h, w) for h, w in SIZES if h * w],
                                                                      eng.DEFAULT_TILE, model._mode()))
    with torch.no_grad():
        outs = model.forward_many(*[list(t) for t in zip(*items)])
        alone = [model(*it) for it in items]
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    assert len(outs) == len(items)
    for i, (o, a) in enumerate(zip(outs, alone)):
        _equal(o, a, f"image {i} {SIZES[i]}")


@pytest.mark.parametrize("precision", ["default", "bf16x3"])
def test_forward_ragged_windows_of_a_large_image(precision):
    """A 1080p image cut into 256-pixel windows beside small images, several passes, channels_last and sliced
    inputs: each image equals the untiled forward of it alone."""
    model = _model(ofw.synthetic_state_dict(5, 3.0), precision).eval()
    mode = model._mode()
    sizes = [(1080, 1920), (37, 53), (300, 520), (1, 1)]
    items = _inputs(sizes, 2, lambda i: i != 2)
    items[0] = tuple(t.contiguous(memory_format=torch.channels_last) for t in items[0])
    items[2] = tuple(torch.cat([t, t], 3)[..., ::2] for t in items[2])  # strided view
    eng = model.engine()
    _poison_forward_workspace(eng, eng.forward_ragged_workspace_bytes(sizes, (256, 256), mode, 300_000))
    with torch.no_grad():
        outs = eng.forward_ragged(items, (256, 256), mode, max_pass_pixels=300_000)
        alone = [eng.forward(*it, mode=mode) for it in items]
    torch.cuda.synchronize()
    assert not eng.f8_overflowed()
    for i, (o, a) in enumerate(zip(outs, alone)):
        _equal(o, a, f"image {i} {sizes[i]}")


def test_forward_many_batched_items_and_fp32_refused():
    model = _model(ofw.synthetic_state_dict(1, 3.0)).eval()
    items = _inputs([(16, 24), (9, 5)], 4, lambda i: False)
    items[0] = tuple(torch.cat([t, t.flip(3)], 0) for t in items[0])  # an item of two images
    with torch.no_grad():
        outs = model.forward_many(*[list(t) for t in zip(*items)])
        for o, it in zip(outs, items):
            _equal(o, model(*it), "item")
    model.precision = "fp32"
    with pytest.raises(ValueError, match="tensor cores"):
        model.forward_many(*[list(t) for t in zip(*items)])


def _per_image_training(eng, items, shapes, grads_out):
    outs, gins, gpars = [], [], []
    for it, g in zip(items, grads_out):
        out, saved = eng.forward_train(*it)
        gp, gi = eng.backward(g, saved, shapes, want_input_grads=True)
        outs.append(out)
        gins.append(gi)
        gpars.append(gp)
    torch.cuda.synchronize()
    return outs, gins, gpars


@pytest.mark.parametrize("sd_kind", ["smooth", "gated"])
@pytest.mark.parametrize("max_pixels", [None, 20000])
def test_train_ragged_matches_per_image(sd_kind, max_pixels):
    """Outputs and input gradients bit for bit against wn_forward_train / wn_backward of each image alone; parameter
    gradients within the float64 bar of the summed references.  max_pixels lowers the engine's grouping limit, so
    the list spans several training calls whose parameter gradients are added in order."""
    sd = (gr.smooth_state_dict if sd_kind == "smooth" else gr.gated_state_dict)(7)
    model = _model(sd)
    eng = model.engine()
    if max_pixels:
        eng.TRAIN_MAX_PIXELS = max_pixels
    _poison_train_workspaces(eng)
    sizes = [s for s in SIZES if s[0] * s[1]]
    items = _inputs(sizes, 9, lambda i: i % 3 == 0)
    g = torch.Generator().manual_seed(1)
    grads_out = [torch.randn((1, 3, h, w), generator=g).cuda() for h, w in sizes]
    shapes = [p.shape for p in model.parameters()]
    outs, saved = eng.forward_train_ragged(items)
    if max_pixels:
        assert len(saved) > 1
    want = [(True,) * 4 for _ in items]
    gpar, gin = eng.backward_ragged(grads_out, saved, shapes, want)
    torch.cuda.synchronize()
    del eng._train_ragged_workspace
    a_out, a_gin, a_gpar = _per_image_training(eng, items, shapes, grads_out)
    for i in range(len(items)):
        _equal(outs[i], a_out[i], f"output of image {i} {sizes[i]}")
        for t in range(4):
            _equal(gin[i][t], a_gin[i][t], f"d/d{gr.INPUT_NAMES[t]} of image {i} {sizes[i]}")
    refs = [gr.reference(sd, it, grad=go, device="cuda") for it, go in zip(items, grads_out)]
    for r in refs:
        gr.assert_relus_cannot_flip(r.z)
    worst = 0.0
    for k, name in enumerate(gr.PARAM_NAMES):
        R = sum(r.grads[name] for r in refs)
        M = sum(r.M[name] for r in refs)
        worst = max(worst, gr.assert_grad_close(gpar[k], R, M, gr.TAU_ONE_PIXEL, name))
        # and against the sum of the per-image gradients of the library itself
        gr.assert_grad_close(gpar[k], sum(p[k].double() for p in a_gpar), M, gr.TAU_ONE_PIXEL, name + " (sum)")
    print(f"worst |G - R| / M: {worst:.3g}")


def test_forward_many_autograd_routes_gradients():
    sd = gr.smooth_state_dict(2)
    model = _model(sd)
    sizes = [(13, 21), (40, 8), (1, 1)]
    items = _inputs(sizes, 3, lambda i: i == 1)
    # item 0: x and gc require grad; item 1: none; item 2: wb
    req = [(True, False, False, True), (False,) * 4, (False, True, False, False)]
    leaves = [tuple(t.clone().requires_grad_(r) for t, r in zip(it, rq)) for it, rq in zip(items, req)]
    outs = model.forward_many(*[list(t) for t in zip(*leaves)])
    loss = sum((o * (k + 1)).square().sum() for k, o in enumerate(outs))
    loss.backward()
    ragged_par = [p.grad.clone() for p in model.parameters()]
    model.zero_grad(set_to_none=True)
    per_in = []
    for k, it in enumerate(items):
        lv = tuple(t.clone().requires_grad_(r) for t, r in zip(it, req[k]))
        ((model(*lv) * (k + 1)).square().sum()).backward()
        per_in.append(lv)
    torch.cuda.synchronize()
    for k in range(len(items)):
        for t in range(4):
            if req[k][t]:
                _equal(leaves[k][t].grad, per_in[k][t].grad, f"item {k} input {t}")
            else:
                assert leaves[k][t].grad is None
    for a, b in zip(ragged_par, model.parameters()):
        torch.testing.assert_close(a, b.grad, rtol=1e-3, atol=1e-3 * b.grad.abs().max().item())


def test_forward_many_params_modified_between_forward_and_backward():
    model = _model(gr.smooth_state_dict(4))
    items = _inputs([(9, 9), (5, 17)], 0, lambda i: False)
    outs = model.forward_many(*[list(t) for t in zip(*items)])
    with torch.no_grad():
        model.cmg.conv1.bias.add_(0.01)
    model.engine()  # repack the edited weights
    with pytest.raises(RuntimeError, match="modified between forward and backward"):
        sum(o.sum() for o in outs).backward()


def test_train_ragged_refuses_an_image_over_the_training_limit():
    from waternet_b200 import _lib
    model = _model(gr.smooth_state_dict(4))
    eng = model.engine()
    eng.TRAIN_MAX_PIXELS = 100
    items = _inputs([(9, 9), (11, 11)], 0, lambda i: False)
    with pytest.raises(_lib.WaterNetLibraryError, match="grad_tile"):
        eng.forward_train_ragged(items)


def test_train_py_native_size_writes_its_artefacts(tmp_path):
    """train.py --synthetic --native-size: mixed sizes through the ragged loader and WaterNet.forward_many."""
    import json
    import os
    import shutil
    import subprocess
    import sys

    from conftest import ROOT
    shutil.copy(os.path.join(ROOT, "train.py"), tmp_path / "train.py")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(ROOT), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, str(tmp_path / "train.py"), "--synthetic", "--native-size", "--epochs", "2",
                          "--height", "64", "--width", "64", "--seed", "0"], cwd=tmp_path, env=env,
                         capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    run = tmp_path / "training" / "0"
    for name in ("last.pt", "metrics-train.csv", "metrics-val.csv", "config.json"):
        assert (run / name).is_file(), name
    assert json.loads((run / "config.json").read_text())["native_size"] is True
    rows = (run / "metrics-train.csv").read_text().strip().splitlines()
    assert len(rows) == 3  # header + 2 epochs
    assert all(np_finite(v) for v in rows[-1].split(","))


def np_finite(v):
    import math
    return math.isfinite(float(v))
