"""tile="auto" / grad_tile="auto" on the GPU: each call takes the path Engine.auto_tile chooses and returns the bits
of the explicit setting of that path, at both sides of the budget; at true size a 45 MP photo runs in windows."""
import gc
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import forward as ofw

pytestmark = pytest.mark.gpu

UNDER, OVER = 1 << 62, 1  # budgets that every call fits / that no call fits
SPIED = ("forward", "forward_tiled", "confidence_maps", "confidence_maps_tiled", "refine", "refine_tiled", "enhance",
         "enhance_tiled", "forward_train", "backward", "backward_tiled", "confidence_maps_train",
         "confidence_maps_backward", "confidence_maps_backward_tiled", "refine_train", "refine_backward",
         "refine_backward_tiled", "forward_ragged", "forward_train_ragged", "backward_ragged", "backward_ragged_tiled",
         "perceptual_loss")


@pytest.fixture
def budget(monkeypatch):
    """Sets Engine.AUTO_WORKSPACE_BYTES for one test (monkeypatch restores it)."""
    from waternet_b200.engine import Engine

    def set_budget(nbytes):
        monkeypatch.setattr(Engine, "AUTO_WORKSPACE_BYTES", nbytes)
    return set_budget


@pytest.fixture
def spy(monkeypatch):
    """The Engine methods called, in order (``perceptual_loss`` as (name, tile))."""
    from waternet_b200.engine import Engine
    calls = []
    for name in SPIED:
        def wrap(self, *args, _orig=getattr(Engine, name), _name=name, **kwargs):
            calls.append((_name, kwargs.get("tile")) if _name == "perceptual_loss" else _name)
            return _orig(self, *args, **kwargs)
        monkeypatch.setattr(Engine, name, wrap)
    return calls


def _model(precision="default", **kw):
    from waternet_b200.net import WaterNet
    m = WaterNet(precision=precision, **kw)
    m.load_state_dict(ofw.synthetic_state_dict(0, 3.0))
    return m.cuda()


def _rand(k, n, h, w, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.rand((n, 3, h, w), generator=g, device="cuda") for _ in range(k)]


def _assert_bitwise(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert a.shape == b.shape, what
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), \
        f"{what}: {int((a != b).sum())} of {a.numel()} values differ"


# ---- inference ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["default", "bf16x3"])
@pytest.mark.parametrize("side", ["under", "over"])
def test_inference_takes_the_path_of_the_budget(budget, spy, precision, side):
    m = _model(precision).eval()
    ins = _rand(4, 2, 96, 128)
    budget(UNDER if side == "under" else OVER)
    sfx = "" if side == "under" else "_tiled"

    def calls():
        return [m(*ins), torch.cat(m.cmg(*ins), 1), m.ce_refiner(ins[0], ins[2])]
    with torch.no_grad():
        m.tile = "auto"
        spy.clear()
        got = calls()
        assert spy == ["forward" + sfx, "confidence_maps" + sfx, "refine" + sfx]
        m.tile = None if side == "under" else 998
        want = calls()
    for g, w, what in zip(got, want, ("model", "cmg", "ce_refiner")):
        _assert_bitwise(g, w, f"{what} {precision} {side}")


@pytest.mark.parametrize("precision", ["default", "bf16x3"])
def test_enhancer_auto_takes_the_path_of_the_budget(budget, spy, precision):
    from waternet_b200.api import Enhancer
    m = _model(precision).eval()
    frames = np.stack([ofw.synthetic_image(i, 96, 128, "noise") for i in range(3)])
    auto = Enhancer(m, tile="auto")
    budget(UNDER)
    spy.clear()
    got = auto(frames)
    assert set(spy) == {"enhance"}
    assert any(s.graph is not None for s in auto._slots)  # the whole-image path keeps its graph capture
    assert np.array_equal(got, Enhancer(m)(frames))
    budget(OVER)
    spy.clear()
    got = auto(frames)
    assert spy == ["enhance_tiled"] * 3  # one image per pipelined pass
    assert np.array_equal(got, Enhancer(m, tile=998)(frames))
    pin = torch.empty(1, 32, 32, 3, dtype=torch.uint8).pin_memory()
    with pytest.raises(ValueError, match="exchange"):
        auto.submit(pin, torch.empty_like(pin).pin_memory(), exchange=object())
    spy.clear()
    whole = Enhancer(m, precision="fp32", tile="auto")(frames)  # no windows in fp32: whole images at any budget
    assert set(spy) == {"enhance"}
    assert np.array_equal(whole, Enhancer(m, precision="fp32")(frames))


def test_45_mp_photo_runs_in_windows_at_the_default_budget(spy):
    from waternet_b200.engine import Engine
    assert Engine.AUTO_WORKSPACE_BYTES is None
    m = _model(tile="auto").eval()
    m.engine().release_workspaces()
    gc.collect()
    torch.cuda.empty_cache()
    ins = _rand(4, 1, 5504, 8256)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        got = m(*ins)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print(f"peak device memory {peak / 1e9:.2f} GB")
    assert spy == ["forward_tiled"]
    assert peak < 20e9
    m.tile = 998
    with torch.no_grad():
        _assert_bitwise(got, m(*ins), "45 MP photo")
    del got, ins
    m.engine().release_workspaces()


# ---- training -----------------------------------------------------------------------------------------------------
def _free_refiner():
    from waternet_b200.net import Refiner
    r = Refiner()
    sd = ofw.synthetic_state_dict(0, 3.0)
    r.load_state_dict({k[len("gc_refiner."):]: v for k, v in sd.items() if k.startswith("gc_refiner.")})
    return r.cuda()


def _many(m, xs):
    return torch.cat([o.flatten() for o in m.forward_many(xs[0::4], xs[1::4], xs[2::4], xs[3::4])])


# kind -> (module factory, call, inputs, methods of the whole-image path, methods of the windowed path)
KINDS = {
    "model": (_model, lambda m, xs: m(*xs), lambda: _rand(4, 2, 64, 80),
              ["forward_train", "backward"], ["forward_tiled", "backward_tiled"]),
    "cmg": (_model, lambda m, xs: torch.cat(m.cmg(*xs), 1), lambda: _rand(4, 2, 64, 80),
            ["confidence_maps_train", "confidence_maps_backward"],
            ["confidence_maps_tiled", "confidence_maps_backward_tiled"]),
    "refiner": (_free_refiner, lambda r, xs: r(*xs), lambda: _rand(2, 2, 64, 80),
                ["refine_train", "refine_backward"], ["refine_tiled", "refine_backward_tiled"]),
    "forward_many": (_model, _many, lambda: _rand(4, 1, 64, 80) + _rand(4, 2, 48, 96, seed=1),
                     ["forward_train_ragged", "backward_ragged"], ["forward_ragged", "backward_ragged_tiled"]),
}


def _gradients(m, call, ins, seed=7):
    """Output, parameter gradients and input gradients of ``call`` under a fixed d(loss)/d(out)."""
    m.zero_grad(set_to_none=True)
    xs = [t.clone().requires_grad_() for t in ins]
    out = call(m, xs)
    g = torch.rand(out.shape, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda")
    out.backward(g)
    return [out.detach()] + [None if p.grad is None else p.grad.clone() for p in m.parameters()] + \
        [x.grad.clone() for x in xs]


@pytest.mark.parametrize("train_precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("side", ["under", "over"])
def test_grad_tile_auto_takes_the_path_of_the_budget(budget, spy, train_precision, kind, side):
    make, call, inputs, whole, windowed = KINDS[kind]
    m = make()
    m.train_precision = train_precision
    ins = inputs()
    budget(UNDER if side == "under" else OVER)
    m.grad_tile = "auto"
    spy.clear()
    got = _gradients(m, call, ins)
    assert spy == (whole if side == "under" else windowed)
    m.grad_tile = None if side == "under" else 998
    want = _gradients(m, call, ins)
    assert len(got) == len(want)
    for k, (a, b) in enumerate(zip(got, want)):
        _assert_bitwise(a, b, f"{kind} {train_precision} {side}: tensor {k}")


def test_an_image_over_the_training_limit_runs_in_windows_with_auto(spy):
    from waternet_b200 import _lib
    m = _model()
    ins = _rand(4, 1, 3000, 3000)
    with pytest.raises(_lib.WaterNetLibraryError, match="exceeds"):
        m(*[t.clone().requires_grad_() for t in ins])
    m.grad_tile = "auto"
    spy.clear()
    got = _gradients(m, KINDS["model"][1], ins)
    assert spy == ["forward_tiled", "backward_tiled"]
    m.grad_tile = 998
    want = _gradients(m, KINDS["model"][1], ins)
    for k, (a, b) in enumerate(zip(got, want)):
        _assert_bitwise(a, b, f"3000 x 3000: tensor {k}")


def test_backward_runs_the_path_its_forward_chose(budget, spy):
    m = _model(grad_tile="auto")
    ins = _rand(4, 2, 64, 80)
    for first, then, path in ((UNDER, OVER, "backward"), (OVER, UNDER, "backward_tiled")):
        budget(first)
        out = m(*[t.clone().requires_grad_() for t in ins])
        budget(then)
        spy.clear()
        out.sum().backward()
        assert spy == [path]


# ---- the VGG loss and the command line ------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["under", "over"])
def test_perceptual_loss_auto_takes_the_path_of_the_budget(budget, spy, side):
    from waternet_b200.engine import Engine
    from waternet_b200.training import PerceptualModel, perceptual_loss
    vgg = PerceptualModel(pretrained=False, native=True, tile="auto").cuda().eval()
    out, ref = _rand(2, 2, 96, 128)
    budget(UNDER if side == "under" else OVER)

    def run(tile):
        vgg.tile = tile
        o = out.clone().requires_grad_()
        loss = perceptual_loss(vgg, o, ref)
        loss.backward()
        return loss.detach(), o.grad

    spy.clear()
    got = run("auto")
    assert spy == [("perceptual_loss", None if side == "under" else Engine.DEFAULT_TILE)]
    want = run(None if side == "under" else 998)
    _assert_bitwise(got[0].reshape(1), want[0].reshape(1), "loss")
    _assert_bitwise(got[1], want[1], "d(out)")


def test_inference_cli_tile_auto_writes_the_same_files(tmp_path):
    import cv2
    shutil.copy(os.path.join(ROOT, "inference.py"), tmp_path / "inference.py")  # it writes under its own output/
    src = tmp_path / "src"
    src.mkdir()
    for i, (h, w) in enumerate(((96, 128), (120, 200), (64, 64))):
        cv2.imwrite(str(src / f"img{i}.png"), ofw.synthetic_image(i, h, w, "noise"))
    torch.save(ofw.synthetic_state_dict(0, 3.0), tmp_path / "w.pt")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(p for p in (ROOT, os.environ.get("PYTHONPATH")) if p))
    for name, extra in (("plain", []), ("auto", ["--tile", "auto"])):
        res = subprocess.run([sys.executable, "inference.py", "--source", "src", "--weights", "w.pt", "--name", name,
                              *extra], cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
        assert res.returncode == 0, res.stderr
    for i in range(3):
        plain = (tmp_path / "output" / "plain" / f"img{i}.png").read_bytes()
        assert plain == (tmp_path / "output" / "auto" / f"img{i}.png").read_bytes(), i
