"""The native SSIM / PSNR (wn_quality, metrics.native_quality) on the GPU, against the float64 restatement of
tests/metrics_reference.py.

The bar.  SSIM of a pixel is formed in fp32 from five fp32 moments.  With exact moments the formula alone rounds
about ten times, each by at most u = 2^-24 of a value of magnitude <= 1: 10 u = 6e-7 in a pixel and so in any
mean of pixels.  The moments add their own error, 22 rounded multiply-adds of the separable window against the 121
of torch's convolution, taken of values centred on the group's mid-range; where the values are far from zero or
nearly constant, torch's E[x^2] - E[x]^2 cancels and the centred moments do not.  So the bar holds native to torch:

    |native - float64| <= 4 max(|torch fp32 - float64|, 6e-7)     for the SSIM of every batch and list,

and to 1e-9 dB for PSNR, whose squared differences and sums are float64 (only the final log10 and division remain).
"""
import os

import numpy as np
import pytest
import torch

import metrics_reference as mref
from waternet_b200 import metrics, training as T

pytestmark = pytest.mark.gpu

SIZES = [(6, 6), (11, 11), (12, 13), (64, 97), (112, 112)]
KINDS = ["noise", "smooth", "flat"]
FLOOR = 6e-7
FACTOR = 4
PSNR_BAR = 1e-9


def _cuda(a):
    return torch.from_numpy(a).cuda()


def _ragged_sizes(count=32, seed=3):
    rng = np.random.default_rng(seed)
    return [(int(rng.integers(6, 300)), int(rng.integers(6, 300))) for _ in range(count)]


def _check(outs, refs):
    """Native against float64 within the bar; returns the SSIM errors of native and of torch fp32."""
    want_s, want_p = mref.quality(outs, refs)
    if isinstance(outs, list):
        got = metrics.native_quality([_cuda(o) for o in outs], [_cuda(r) for r in refs])
        torch_s = T.batch_quality([_cuda(o) for o in outs], [_cuda(r) for r in refs])[0].item()
    else:
        got = metrics.native_quality(_cuda(outs), _cuda(refs))
        torch_s = metrics.ssim(_cuda(outs), _cuda(refs)).item()
    s, p = (v.item() for v in got)
    assert got[0].dim() == 0 and got[0].is_cuda and got[1].dim() == 0
    err, terr = abs(s - want_s), abs(torch_s - want_s)
    assert err <= FACTOR * max(terr, FLOOR), f"SSIM {s} vs float64 {want_s}: {err:.3g} (torch fp32 {terr:.3g})"
    assert abs(p - want_p) <= PSNR_BAR, f"PSNR {p} vs float64 {want_p}"
    return err, terr


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_batch_against_float64(size, kind):
    _check(*mref.inputs(kind, (4, 3, *size), seed=size[1]))


@pytest.mark.parametrize("kind", KINDS)
def test_list_against_float64(kind):
    pairs = [mref.inputs(kind, (1 + k % 2, 3, *s), seed=k) for k, s in enumerate(SIZES)]
    _check([o for o, _ in pairs], [r for _, r in pairs])


@pytest.mark.parametrize("kind", KINDS)
def test_1080p_against_float64(kind):
    _check(*mref.inputs(kind, (2, 3, 1080, 1920), seed=7))


@pytest.mark.parametrize("kind", KINDS)
def test_ragged_list_of_32_sizes_against_float64(kind):
    pairs = [mref.inputs(kind, (1, 3, h, w), seed=k) for k, (h, w) in enumerate(_ragged_sizes())]
    _check([o for o, _ in pairs], [r for _, r in pairs])


def _network_outputs():
    """Outputs of the trained golden weights on smooth synthetic images, and those images as references."""
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


def test_network_outputs_against_float64():
    out, ref = _network_outputs()
    _check(out, ref)
    _check([out[:1], out[1:]], [ref[:1], ref[1:]])


@pytest.mark.parametrize("value", [0.0, 0.25, 0.3, 1.0])
def test_constant_pair_gives_nan_without_fault(value):
    a = torch.full((2, 3, 16, 16), value, device="cuda")
    s, p = metrics.native_quality(a, a)
    assert torch.isnan(s) and torch.isinf(p)
    s, _ = metrics.native_quality([a[:1], torch.rand(1, 3, 20, 20, device="cuda")], [a[:1], torch.rand(1, 3, 20, 20, device="cuda")])
    assert torch.isnan(s)
    b = torch.full_like(a, value / 2 + 0.1)  # two different constants: data range 0 as well, c1 = c2 = 0
    s, p = metrics.native_quality(a, b)
    torch.cuda.synchronize()
    assert torch.isfinite(p)


def _stats(outs, refs, groups):
    from waternet_b200.engine import get_engine
    return get_engine("cuda:0").quality(outs, refs, groups)


def test_image_of_a_list_equals_the_image_alone_bit_for_bit():
    pairs = [mref.inputs("noise", (1, 3, h, w), seed=k) for k, (h, w) in enumerate(_ragged_sizes())]
    outs, refs = [_cuda(o)[0] for o, _ in pairs], [_cuda(r)[0] for _, r in pairs]
    together = _stats(outs, refs, list(range(len(outs))))
    for i in (0, 7, 31):
        alone = _stats([outs[i]], [refs[i]], [0])
        assert torch.equal(together[i].view(torch.int64), alone[0].view(torch.int64)), i
    # a group of a batch: the group's statistics do not depend on other groups in the call
    both = _stats(outs[:3] + outs[3:5], refs[:3] + refs[3:5], [1, 1, 1, 0, 0])
    first = _stats(outs[:3], refs[:3], [0, 0, 0])
    assert torch.equal(both[:3].view(torch.int64), first.view(torch.int64))


def test_repeated_calls_are_bit_identical():
    o, r = (_cuda(a) for a in mref.inputs("noise", (4, 3, 1080, 1920), seed=1))
    first = torch.stack(metrics.native_quality(o, r))
    for _ in range(3):
        assert torch.equal(torch.stack(metrics.native_quality(o, r)).view(torch.int64), first.view(torch.int64))


def test_peak_memory_is_the_workspace_plus_a_few_mb():
    from waternet_b200.engine import get_engine
    eng = get_engine("cuda:0")
    o, r = (_cuda(a) for a in mref.inputs("noise", (4, 3, 1080, 1920), seed=2))
    eng.release_workspaces()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    metrics.native_quality(o, r)
    torch.cuda.synchronize()
    grown = torch.cuda.max_memory_allocated() - base
    ws = eng.quality_workspace_bytes([(1080, 1920)] * 4)
    assert grown <= ws + (4 << 20), (grown, ws)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.max_memory_allocated()
    T.batch_quality(o, r)
    torch.cuda.synchronize()
    torch_grown = torch.cuda.max_memory_allocated() - base
    print(f"\n4 x 1080p: native grows {grown / 2**20:.1f} MiB (workspace {ws / 2**20:.2f} MiB), "
          f"torch {torch_grown / 2**20:.0f} MiB ({torch_grown / o[:, 0].numel():.0f} B per pixel)")
    assert torch_grown > 50 * grown


def _train(tmp_path, metrics_value):
    import shutil
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    work = tmp_path / metrics_value
    work.mkdir()
    for f in ("train.py",):
        shutil.copy(os.path.join(root, f), work / f)
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run([sys.executable, "train.py", "--synthetic", "--epochs", "1", "--batch-size", "16",
                          "--seed", "0", "--perceptual", "native", "--metrics", metrics_value], cwd=work, env=env, capture_output=True,
                         text=True, timeout=1800)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    run = work / "training" / "0"
    import json
    assert json.loads((run / "config.json").read_text())["metrics"] == metrics_value
    rows = {}
    for name in ("train", "val"):
        lines = (run / f"metrics-{name}.csv").read_text().splitlines()
        rows[name] = dict(zip(lines[0].split(","), map(float, lines[1].split(","))))
    return rows


def test_train_py_with_native_metrics_agrees_with_torch(tmp_path):
    """The SSIM / PSNR columns of a --metrics native run against a --metrics torch run of the same seed.  The training
    (native perceptual loss, deterministic) is the same in both, so the loss columns are equal; the metric columns
    differ by torch fp32's error and native's (the bar: at most 4 times torch's, with torch's about 1e-6 on these
    images), plus the six decimals of the files' "%f"."""
    a, b = _train(tmp_path, "torch"), _train(tmp_path, "native")
    for split in ("train", "val"):
        for col, tol in (("ssim", 2e-5), ("psnr", 1e-4)):
            assert abs(a[split][col] - b[split][col]) <= tol, (split, col, a[split][col], b[split][col])
        assert a[split]["mse"] == b[split]["mse"], split
