"""The native SSIM loss (wn_ssim_grad, metrics.ssim_loss) on the GPU: d(out) element by element against the float64
restatement of tests/ssim_grad_reference.py within its bar (4 max(torch fp32's worst error, F), DESIGN.md 4.17), the
statistics and the loss against wn_quality bit for bit, ragged and repeated calls bit for bit, WaterNet's parameter
gradients against torch autograd of metrics.ssim, no_grad, and train.py --ssim-weight."""
import os

import numpy as np
import pytest
import torch

import metrics_reference as mref
import ssim_grad_reference as sgr
from waternet_b200 import metrics, training as T

pytestmark = pytest.mark.gpu

SIZES = [(6, 6), (8, 40), (10, 10), (11, 11), (12, 13), (64, 97)]
KINDS = ["noise", "smooth", "flat"]


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _torch32(out, ref):
    """torch fp32 autograd of 1 - ssim (1 - batch_quality(...)[0] for lists) on the CPU, where no TF32 applies."""
    if isinstance(out, list):
        to = [torch.from_numpy(o).requires_grad_() for o in out]
        s = T.batch_quality(to, [torch.from_numpy(r) for r in ref])[0]
        return [g.numpy() for g in torch.autograd.grad(1 - s, to)]
    to = torch.from_numpy(out).requires_grad_()
    return torch.autograd.grad(1 - metrics.ssim(to, torch.from_numpy(ref)), to)[0].numpy()


def _native(out, ref):
    """(loss, d(out)) of ssim_loss through autograd."""
    if isinstance(out, list):
        to = [_cuda(o).requires_grad_() for o in out]
        loss = metrics.ssim_loss(to, [_cuda(r) for r in ref])
        loss.backward()
        return loss, [t.grad.cpu().numpy() for t in to]
    to = _cuda(out).requires_grad_()
    loss = metrics.ssim_loss(to, _cuda(ref))
    loss.backward()
    return loss, to.grad.cpu().numpy()


def _check(out, ref, floor_only=False):
    """d(out) within the bar; ``floor_only``: within 4 F alone, where torch fp32's error is no yardstick (nearly
    constant images: its uncentred moments cancel)."""
    loss, got = _native(out, ref)
    assert loss.dim() == 0 and loss.dtype == torch.float32 and loss.is_cuda
    want, m = sgr.grad(out, ref, terms=True)
    bad, worst, allowed = sgr.bar_violations(got, want, _torch32(out, ref), m)
    assert bad == 0, f"{bad} elements beyond the bar: worst {worst:.3g} > {allowed:.3g}"
    assert not floor_only or worst <= sgr.FACTOR * sgr.floor(m), (worst, sgr.FACTOR * sgr.floor(m))
    print(f"\n|G - R| <= {worst:.3g}, bar {allowed:.3g} (floor {sgr.FACTOR * sgr.floor(m):.3g})")
    return worst, allowed


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_batch_against_float64(size, kind):
    for n in (1, 3):
        _check(*mref.inputs(kind, (n, 3, *size), seed=size[1] + n), floor_only=kind == "flat")


@pytest.mark.parametrize("kind", KINDS)
def test_list_against_float64(kind):
    pairs = [mref.inputs(kind, (1 + k % 3, 3, *s), seed=k) for k, s in enumerate(SIZES)]
    _check([o for o, _ in pairs], [r for _, r in pairs], floor_only=kind == "flat")


@pytest.mark.parametrize("kind", KINDS)
def test_1080p_against_float64(kind):
    _check(*mref.inputs(kind, (1, 3, 1080, 1920), seed=7), floor_only=kind == "flat")


def test_batch_of_130x70_against_float64():
    _check(*mref.inputs("noise", (2, 3, 130, 70), seed=5))
    r, o = mref.inputs("noise", (2, 3, 130, 70), seed=6)  # out the clipped one: ties at 0 and 1, its range larger
    _check(o, r)


def _ragged_sizes(count=32, seed=3):
    rng = np.random.default_rng(seed)
    return [(int(rng.integers(6, 300)), int(rng.integers(6, 300))) for _ in range(count)]


@pytest.mark.parametrize("kind", ["noise", "smooth"])
def test_ragged_list_of_32_sizes_against_float64(kind):
    pairs = [mref.inputs(kind, (1, 3, h, w), seed=k) for k, (h, w) in enumerate(_ragged_sizes())]
    _check([o for o, _ in pairs], [r for _, r in pairs])


def _network_outputs():
    """Outputs of the trained golden weights (ReLU ties at 0) and their inputs as references."""
    from oracle import forward as ofw
    from waternet_b200.engine import get_engine
    from waternet_b200.net import WaterNet
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trained_synthetic_400ep.npz")
    with np.load(path) as z:
        sd = {k: torch.from_numpy(z[k]) for k in z.files}
    model = WaterNet()
    model.load_state_dict(sd)
    model = model.cuda().eval()
    rgb = np.stack([ofw.synthetic_image(s, 96, 128, "smooth") for s in range(3)])
    res = get_engine("cuda:0").preprocess(torch.from_numpy(rgb).cuda(), tensors=True)
    with torch.no_grad():
        out = model(res["x"], res["wb"], res["he"], res["gc"])
    return out.cpu().numpy(), res["x"].cpu().numpy()


def test_network_outputs_with_ties_against_float64():
    out, ref = _network_outputs()
    _check(out, ref)
    _check([out[:1], out[1:]], [ref[:1], ref[1:]])
    o, r = out.copy(), ref.copy()
    o[:, :, :20] = 0.0  # a ReLU's zeros: many ties at the minimum
    assert (o == o.min()).sum() > 1000
    _check(o, r)


def _stats_call(outs, refs, groups, scales):
    from waternet_b200.engine import get_engine
    return get_engine("cuda:0").ssim_grad(outs, refs, groups, scales)


def _bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int64)


def test_stats_and_loss_equal_wn_quality_bit_for_bit():
    from waternet_b200.engine import get_engine
    for shape in [(4, 3, 64, 97), (2, 3, 8, 40), (1, 3, 1080, 1920)]:
        o, r = (_cuda(a) for a in mref.inputs("noise", shape, seed=1))
        stats, _ = _stats_call(list(o), list(r), [0] * len(o), [1.0] * len(o))
        want = get_engine("cuda:0").quality(list(o), list(r), [0] * len(o))
        assert torch.equal(_bits(stats), _bits(want)), shape
        leaf = o.clone().requires_grad_()
        loss = metrics.ssim_loss(leaf, r)
        assert torch.equal(_bits(loss), _bits((1.0 - metrics.native_quality(o, r)[0]).float())), shape
    pairs = [mref.inputs("smooth", (1 + k % 2, 3, *s), seed=k) for k, s in enumerate(SIZES)]
    lo, lr = [_cuda(a).requires_grad_() for a, _ in pairs], [_cuda(b) for _, b in pairs]
    loss = metrics.ssim_loss(lo, lr)
    assert torch.equal(_bits(loss), _bits((1.0 - metrics.native_quality([t.detach() for t in lo], lr)[0]).float()))


def test_image_of_a_ragged_call_equals_the_image_alone_and_calls_repeat_bit_for_bit():
    pairs = [mref.inputs("noise", (1, 3, h, w), seed=k) for k, (h, w) in enumerate(_ragged_sizes())]
    outs, refs = [_cuda(o)[0] for o, _ in pairs], [_cuda(r)[0] for _, r in pairs]
    n = len(outs)
    scales = [-1.0 / n] * n
    stats, grads = _stats_call(outs, refs, list(range(n)), scales)
    for i in (0, 7, 31):
        s1, g1 = _stats_call([outs[i]], [refs[i]], [0], [scales[i]])
        assert torch.equal(_bits(stats[i]), _bits(s1[0])), i
        assert torch.equal(_bits(grads[i]), _bits(g1[0])), i
    # a group of a batch against the same group alone in another call
    both_s, both_g = _stats_call(outs[:3] + outs[3:5], refs[:3] + refs[3:5], [1, 1, 1, 0, 0], [0.5] * 5)
    s3, g3 = _stats_call(outs[:3], refs[:3], [0, 0, 0], [0.5] * 3)
    assert torch.equal(_bits(both_s[:3]), _bits(s3))
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(both_g[:3], g3))
    for _ in range(2):
        s2, g2 = _stats_call(outs, refs, list(range(n)), scales)
        assert torch.equal(_bits(stats), _bits(s2))
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(grads, g2))


def test_constant_pair_gives_nan_without_fault():
    a = torch.full((2, 3, 16, 16), 0.25, device="cuda", requires_grad=True)
    loss = metrics.ssim_loss(a, a.detach())
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isnan(loss) and torch.isnan(a.grad).all()


def test_nothing_is_saved_or_written_under_no_grad():
    from waternet_b200.engine import get_engine
    eng = get_engine("cuda:0")
    eng.release_workspaces()
    o = torch.rand(2, 3, 64, 64, device="cuda", requires_grad=True)
    r = torch.rand(2, 3, 64, 64, device="cuda")
    before = eng.launch_count
    with torch.no_grad():
        loss = metrics.ssim_loss(o, r)
    assert loss.grad_fn is None and not loss.requires_grad
    assert eng.launch_count - before == 2  # wn_quality's two launches
    assert "ssim_grad" not in eng._ws
    loss = metrics.ssim_loss(o.detach(), r)  # no out requires grad
    assert loss.grad_fn is None and "ssim_grad" not in eng._ws
    loss = metrics.ssim_loss(o, r)
    assert loss.grad_fn is not None and eng.launch_count - before == 8


def _param_grads(model, loss_fn, *inputs):
    model.zero_grad(set_to_none=True)
    loss_fn(*inputs).backward()
    return [p.grad.clone() for p in model.parameters()]


def _assert_params_close(native, torch_):
    for a, b in zip(native, torch_):
        torch.testing.assert_close(a, b, rtol=1e-3, atol=1e-3 * b.abs().max().item())


@pytest.mark.parametrize("grad_tile", [None, 64])
def test_waternet_parameter_gradients_match_torch_autograd_of_ssim(grad_tile):
    """mse + 0.5 ssim_loss against mse + 0.5 (1 - metrics.ssim) under torch autograd, the same native forward; the
    bar of the other WaterNet backward checks.  grad_tile=64 runs the windowed backward."""
    import grad_reference as gr
    from waternet_b200.net import WaterNet
    torch.backends.cudnn.allow_tf32 = False
    model = WaterNet()
    model.load_state_dict(gr.smooth_state_dict(5))
    model = model.cuda().train()
    model.grad_tile = grad_tile
    g = torch.Generator().manual_seed(3)
    ins = [torch.rand((2, 3, 130, 70), generator=g).cuda() for _ in range(4)]
    ref = torch.rand((2, 3, 130, 70), generator=g).cuda()

    def loss(native):
        out = model(*ins)
        s = metrics.ssim_loss(out, ref) if native else 1 - metrics.ssim(out, ref)
        return torch.mean(torch.square(out - ref)) + 0.5 * s

    _assert_params_close(_param_grads(model, lambda: loss(True)), _param_grads(model, lambda: loss(False)))


def test_forward_many_parameter_gradients_match_torch_autograd_of_batch_quality():
    import grad_reference as gr
    from waternet_b200.net import WaterNet
    torch.backends.cudnn.allow_tf32 = False
    model = WaterNet()
    model.load_state_dict(gr.smooth_state_dict(6))
    model = model.cuda().train()
    g = torch.Generator().manual_seed(4)
    sizes = [(40, 56), (33, 17), (64, 64)]
    items = [[torch.rand((1, 3, h, w), generator=g).cuda() for _ in range(4)] for h, w in sizes]
    refs = [torch.rand((1, 3, h, w), generator=g).cuda() for h, w in sizes]

    def loss(native):
        outs = model.forward_many(*[list(t) for t in zip(*items)])
        s = metrics.ssim_loss(outs, refs) if native else 1 - T.batch_quality(outs, refs)[0]
        return sum(torch.mean(torch.square(o - r)) for o, r in zip(outs, refs)) + 0.5 * s

    _assert_params_close(_param_grads(model, lambda: loss(True)), _param_grads(model, lambda: loss(False)))


def test_train_py_with_ssim_weight_writes_its_artefacts(tmp_path):
    import json
    import shutil
    import subprocess
    import sys
    from conftest import ROOT
    shutil.copy(os.path.join(ROOT, "train.py"), tmp_path / "train.py")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(ROOT), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "train.py", "--synthetic", "--epochs", "1", "--ssim-weight", "0.5",
                          "--seed", "0", "--perceptual", "native"], cwd=tmp_path, env=env, capture_output=True,
                         text=True, timeout=1800)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    run = tmp_path / "training" / "0"
    for name in ("last.pt", "metrics-train.csv", "metrics-val.csv", "config.json"):
        assert (run / name).is_file(), name
    assert json.loads((run / "config.json").read_text())["ssim_weight"] == 0.5
    rows = (run / "metrics-train.csv").read_text().strip().splitlines()
    assert len(rows) == 2 and all(np.isfinite(float(v)) for v in rows[-1].split(","))
