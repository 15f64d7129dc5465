"""tile="auto" / grad_tile="auto" without a GPU: the rule of Engine.auto_tile against the library's own workspace
queries, the handling of the setting on every entry point, and the command lines."""
import argparse
import copy
import io
import json
import pickle
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

GB40 = 40 << 30
P1080 = (1080, 1920)


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


@pytest.fixture
def budget(monkeypatch):
    """Sets Engine.AUTO_WORKSPACE_BYTES for one test (monkeypatch restores it)."""
    from waternet_b200.engine import Engine

    def set_budget(nbytes):
        monkeypatch.setattr(Engine, "AUTO_WORKSPACE_BYTES", nbytes)
    return set_budget


def _auto(kind, shapes, mode=-1, train_mode=None):
    from waternet_b200.engine import Engine
    return Engine.auto_tile(kind, shapes, mode, train_mode)


def test_inference_4k_is_whole_and_8k_is_windowed(lib, budget):
    from waternet_b200.engine import Engine
    budget(GB40)
    for mode in (-1, 1, 2):
        want = lib.wn_forward_workspace_bytes(1, 2160, 3840, mode)
        assert Engine.whole_image_bytes("net", (1, 2160, 3840), mode) == want
        assert _auto("net", (1, 2160, 3840), mode) is None
        assert _auto("net", (16, *P1080), mode) is None  # bench.py's workload: passes of at most 8 Mi pixels
        assert _auto("net", (1, 4320, 7680), mode) == Engine.DEFAULT_TILE
        assert _auto("net", (1, 5504, 8256), mode) == Engine.DEFAULT_TILE  # 45 MP: 84.9 GB
        assert _auto("net", (1, 4000, 6000), mode) == Engine.DEFAULT_TILE  # 24 MP: 44.8 GB
        assert _auto("enhance", (1, 2160, 3840), mode) is None
        assert _auto("enhance", (1, 4320, 7680), mode) == Engine.DEFAULT_TILE


@pytest.mark.parametrize("kind,query", [("net", "wn_forward_workspace_bytes"), ("cmg", "wn_submodule_workspace_bytes"),
                                        ("refiner", "wn_submodule_workspace_bytes"),
                                        ("enhance", "wn_enhance_workspace_bytes")])
def test_a_budget_equal_to_the_call_picks_whole_images(lib, budget, kind, query):
    from waternet_b200.engine import Engine
    need = getattr(lib, query)(3, 720, 1280, -1)
    assert need > 0 and Engine.whole_image_bytes(kind, (3, 720, 1280), -1) == need
    budget(need)
    assert _auto(kind, (3, 720, 1280)) is None
    budget(need - 1)
    assert _auto(kind, (3, 720, 1280)) == Engine.DEFAULT_TILE


def test_training_keeps_every_slice(lib, budget):
    from waternet_b200.engine import Engine
    budget(GB40)
    assert _auto("net", (3, *P1080), train_mode=1) is None
    assert _auto("net", (4, *P1080), train_mode=1) == Engine.DEFAULT_TILE
    assert _auto("net", (16, 112, 112), train_mode=3) is None
    # 9 images of 1080p run as slices of 4, 4 and 1, all kept until backward
    want = 2 * lib.wn_train_workspace_bytes(4, *P1080) + lib.wn_train_workspace_bytes(1, *P1080)
    assert Engine.whole_image_bytes("net", (9, *P1080), -1, 1) == want
    budget(want)
    assert _auto("net", (9, *P1080), train_mode=1) is None
    budget(want - 1)
    assert _auto("net", (9, *P1080), train_mode=1) == Engine.DEFAULT_TILE


def test_an_image_the_training_call_refuses_takes_windows(lib, budget):
    from waternet_b200.engine import Engine
    budget(1 << 62)
    assert 3000 * 3000 > Engine.TRAIN_MAX_PIXELS
    for kind in ("net", "cmg", "refiner"):
        assert Engine.whole_image_bytes(kind, (1, 3000, 3000), -1, 1) == 0
        assert _auto(kind, (1, 3000, 3000), train_mode=1) == Engine.DEFAULT_TILE
        assert _auto(kind, (1, 3000, 3000)) is None  # inference has no such limit
    assert _auto("ragged", [(64, 64), (3000, 3000)], train_mode=1) == Engine.DEFAULT_TILE


def test_a_ragged_list_sums_its_training_calls(lib, budget):
    from waternet_b200.engine import Engine, _sizes, ragged_train_calls
    sizes = [(1080, 1920), (720, 1280), (0, 64), (1080, 1920), (480, 640), (2000, 3000), (64, 96)]
    real = [s for s in sizes if s[0] * s[1]]
    calls = ragged_train_calls(real, Engine.TRAIN_MAX_PIXELS)
    assert len(calls) > 1
    want = sum(lib.wn_train_ragged_workspace_bytes(*_sizes([real[k] for k in idx]), len(idx)) for idx in calls)
    assert Engine.whole_image_bytes("ragged", sizes, -1, 1) == want
    budget(want)
    assert _auto("ragged", sizes, train_mode=1) is None
    budget(want - 1)
    assert _auto("ragged", sizes, train_mode=3) == Engine.DEFAULT_TILE


@pytest.mark.parametrize("kind,stack", [("cmg", 0), ("refiner", 1)])
def test_each_stack_uses_its_own_training_workspace(lib, budget, kind, stack):
    from waternet_b200.engine import Engine
    n, h, w = 6, *P1080  # slices of 4 and 2
    want = (lib.wn_submodule_train_workspace_bytes(4, h, w, stack) +
            lib.wn_submodule_train_workspace_bytes(2, h, w, stack))
    assert Engine.whole_image_bytes(kind, (n, h, w), -1, 1) == want
    assert want < Engine.whole_image_bytes("net", (n, h, w), -1, 1)
    budget(want)
    assert _auto(kind, (n, h, w), train_mode=1) is None
    budget(want - 1)
    assert _auto(kind, (n, h, w), train_mode=1) == Engine.DEFAULT_TILE


def test_the_vgg_loss_takes_one_window_per_image_where_it_fits(lib, budget):
    from waternet_b200.engine import Engine
    need = lib.wn_perceptual_loss_workspace_bytes(4, *P1080, 0, 0, 0)
    assert need > 0 and Engine.whole_image_bytes("vgg", (4, *P1080), 1) == need
    budget(need)
    assert _auto("vgg", (4, *P1080), 1) is None
    budget(need - 1)
    assert _auto("vgg", (4, *P1080), 3) == Engine.DEFAULT_TILE
    budget(1 << 62)
    assert lib.wn_perceptual_loss_workspace_bytes(1, 3000, 3000, 0, 0, 0) == 0  # a window over 8 Mi pixels
    assert _auto("vgg", (1, 3000, 3000), 1) == Engine.DEFAULT_TILE


def test_fp32_and_empty_calls_are_whole_images(lib, budget):
    budget(0)
    for kind in ("net", "cmg", "refiner", "enhance"):
        for train_mode in (None, 1):
            assert _auto(kind, (1, 5504, 8256), 0, train_mode) is None
            assert _auto(kind, (0, 64, 64), -1, train_mode) is None
            assert _auto(kind, (2, 0, 64), -1, train_mode) is None
    assert _auto("ragged", [(5504, 8256)], 0, 1) is None
    assert _auto("ragged", [(0, 8), (8, 0)], -1, 1) is None


def test_unknown_kind_is_refused(lib):
    with pytest.raises(ValueError, match="kind"):
        _auto("vgg19", (1, 64, 64))


# ---- the setting ------------------------------------------------------------------------------------------------
def test_auto_is_accepted_everywhere():
    from waternet_b200.net import ConfidenceMapGenerator, Refiner, WaterNet
    from waternet_b200.training import PerceptualModel
    for precision in ("default", "bf16x3", "fp32"):  # fp32 has no windows: "auto" means whole images there
        m = WaterNet(precision=precision, tile="auto", grad_tile="auto")
        assert m.tile == m.grad_tile == "auto"
        for s in (m.cmg, m.wb_refiner, m.ce_refiner, m.gc_refiner):
            assert s._tile() == s._grad_tile() == "auto" and s.tile is None  # bound stacks follow the parent
    for cls in (ConfidenceMapGenerator, Refiner):
        s = cls()
        s.tile = s.grad_tile = "auto"
        assert s._tile() == s._grad_tile() == "auto"
    assert PerceptualModel(pretrained=False, native=True, tile="auto").tile == "auto"


@pytest.mark.parametrize("bad", ["Auto", "yes", "", "998"])
def test_other_strings_are_refused(bad):
    from waternet_b200.net import Refiner, WaterNet
    from waternet_b200.training import PerceptualModel
    with pytest.raises(ValueError, match="auto"):
        WaterNet(tile=bad)
    with pytest.raises(ValueError, match="auto"):
        WaterNet(grad_tile=bad)
    with pytest.raises(ValueError, match="auto"):
        WaterNet(precision="fp32", tile=bad)
    with pytest.raises(ValueError, match="auto"):
        PerceptualModel(pretrained=False, native=True, tile=bad)
    r = Refiner()
    r.tile = bad
    x = torch.rand(1, 3, 8, 8)
    with torch.no_grad(), pytest.raises(ValueError, match="auto"):
        r(x, x)
    r.tile, r.grad_tile = None, bad
    with pytest.raises(ValueError, match="auto"):
        r(x.requires_grad_(), x)


def test_cpu_tensors_keep_the_torch_graph_with_auto():
    from oracle import forward as ofw
    from waternet_b200.net import Refiner
    sd = ofw.synthetic_state_dict(3, 3.0)
    free = Refiner()
    free.tile = free.grad_tile = "auto"
    free.load_state_dict({k[len("gc_refiner."):]: v for k, v in sd.items() if k.startswith("gc_refiner.")})
    x, gc = (torch.rand(2, 3, 9, 11, generator=torch.Generator().manual_seed(i)) for i in range(2))
    out = free(x, gc)
    assert type(out.grad_fn).__name__ == "ReluBackward0"


def test_auto_survives_deepcopy_and_pickling_and_old_pickles_load_as_none():
    from waternet_b200.net import Refiner, WaterNet
    from waternet_b200.training import PerceptualModel
    net = WaterNet(tile="auto", grad_tile="auto")
    twin = copy.deepcopy(net)
    assert twin.tile == twin.grad_tile == "auto" and twin.gc_refiner._grad_tile() == "auto"
    buf = io.BytesIO()
    torch.save(net, buf)
    buf.seek(0)
    again = torch.load(buf, weights_only=False)
    assert again.tile == again.grad_tile == "auto" and again.cmg._tile() == "auto"
    del again.__dict__["tile"], again.__dict__["grad_tile"]  # a model pickled before the attributes existed
    assert again.tile is None and again.grad_tile is None and again.cmg._tile() is None
    free = Refiner()
    free.grad_tile = "auto"
    back = pickle.loads(pickle.dumps(free))
    assert back.grad_tile == "auto" and copy.deepcopy(free).grad_tile == "auto"
    del back.__dict__["grad_tile"]
    assert back._grad_tile() is None
    vgg = PerceptualModel(pretrained=False, native=True, tile="auto")
    assert pickle.loads(pickle.dumps(vgg)).tile == "auto" and copy.deepcopy(vgg).tile == "auto"


def test_the_perceptual_model_resolves_auto_per_call(lib, budget):
    from waternet_b200.engine import Engine
    from waternet_b200.training import PerceptualModel
    vgg = PerceptualModel(pretrained=False, native=True, tile="auto")
    out = torch.empty(4, 3, *P1080, device="meta")
    need = lib.wn_perceptual_loss_workspace_bytes(4, *P1080, 0, 0, 0)
    budget(need)
    assert vgg._loss_tile(out) is None
    budget(need - 1)
    assert vgg._loss_tile(out) == Engine.DEFAULT_TILE
    vgg.tile = 512
    assert vgg._loss_tile(out) == 512


# ---- command lines ----------------------------------------------------------------------------------------------
def _perceptual_args(*argv):
    from waternet_b200 import training as T
    ap = argparse.ArgumentParser()
    T.add_perceptual_args(ap)
    return ap.parse_args(list(argv))


def test_perceptual_tile_accepts_auto(tmp_path):
    from waternet_b200 import training as T
    args = _perceptual_args("--perceptual", "native", "--perceptual-tile", "auto")
    assert args.perceptual_tile == "auto"
    assert _perceptual_args("--perceptual-tile", "998").perceptual_tile == 998
    T.save_metrics(tmp_path, None, None, {"epochs": 1, **T.perceptual_config(args)})
    assert json.loads((tmp_path / "config.json").read_text())["perceptual_tile"] == "auto"  # the string, not a tile
    with pytest.raises(SystemExit, match="needs --perceptual native"):
        T.perceptual_model(_perceptual_args("--perceptual-tile", "auto"))
    with pytest.raises(SystemExit):
        _perceptual_args("--perceptual-tile", "Auto")


def _run(script, *argv):
    return subprocess.run([sys.executable, script, *argv], cwd=ROOT, capture_output=True, text=True, timeout=300)


def test_the_scripts_parse_auto():
    # each command stops at a check that follows parse_args, so nothing runs on a device
    res = _run("inference.py", "--tile", "auto", "--batch", "0")
    assert "--batch must be at least 1" in res.stderr, res.stderr
    res = _run("train.py", "--grad-tile", "auto", "--perceptual", "native", "--perceptual-tile", "auto",
               "--native-size", "--loader", "torch")
    assert "--native-size needs --loader gpu" in res.stderr, res.stderr
    res = _run("score.py", "--perceptual", "native", "--perceptual-tile", "auto")
    assert "No weights specified" in res.stderr, res.stderr
    for script, flag in (("inference.py", "--tile"), ("train.py", "--grad-tile"), ("score.py", "--perceptual-tile")):
        res = _run(script, flag, "Auto")
        assert res.returncode == 2 and "expected 'auto' or an integer" in res.stderr, (script, res.stderr)
        assert "auto" in _run(script, "--help").stdout
