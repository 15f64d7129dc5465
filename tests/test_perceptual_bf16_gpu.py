"""The single-pass bf16 VGG arithmetic of the native perceptual loss on the GPU (PerceptualModel(precision="bf16"),
the VGG handle in WN_MODE_BF16): every launch replayed in float64 from the GPU's own decoded input, the loss from the
GPU's own features, windows, determinism, mode isolation, autograd, buffer bounds and training.

Bars, measured on an H100 80GB HBM3 (700 W limit); DESIGN.md 4.14.  Per launch the replay bar acc_tau(K) M + 2^-8 |R|
of test_perceptual_bf16_cpu (K = cinpad x 9 forward, the forward cout x 9 for a data gradient), and every decoded
plane exactly bf16; the worst (|G - R| - F) / M measured 2.0e-7 forward, 2.1e-7 backward and 0 for the seed, against
bars of 1.3e-6 (conv1_1) and more.
SEAM_GRAD_REL: 4x the worst norm-wise difference of the windowed d(out) from the one-window d(out), 8.1e-3 (tile 128).
  Not the order of fp32 sums: each window rounds its own share of the halo gradients to bf16 at every launch.
TRAIN_REL: 4x the worst relative difference of the 3-epoch rows between the bf16 and the bf16x3 VGG, 1.47e-3, and
  never looser than the 5 % of tests/train_parity_bf16.sh.
"""
import os

import numpy as np
import pytest
import torch

import buffer_bounds as bb
import test_perceptual_bf16_cpu as vr
import vgg_reference as V
from test_buffer_bounds_gpu import _ok, _outputs, _run

pytestmark = pytest.mark.gpu

SEAM_GRAD_REL = 3.3e-2
TRAIN_REL = 5.9e-3
FOLD_TAU = 2.0 ** -22  # d(out) of one window: one fp32 division of the decoded gradient by std
SHAPES = [(1, 16, 16), (1, 17, 31), (1, 113, 117), (1, 300, 500), (3, 64, 80)]


def _modes():
    from waternet_b200 import _lib
    return _lib.MODE_BF16, _lib.MODE_BF16X3


def _vgg(seed=1234, precision="bf16"):
    from waternet_b200.training import PerceptualModel
    torch.manual_seed(seed)
    return PerceptualModel(pretrained=False, native=True, precision=precision).cuda().eval()


def _pair(n, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = torch.rand((n, 3, h, w), generator=g)
    ref = (out + 0.3 * (torch.rand((n, 3, h, w), generator=g) - 0.5)).clamp(0, 1)
    return out.cuda(), ref.cuda()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def _report(name, value):
    """With WN_REPORT set to a file name: append the measured value (how the bars above were set)."""
    path = os.environ.get("WN_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(f"bf16 {name} {value:.3e}\n")


@pytest.fixture(scope="module")
def vgg():
    return _vgg()


def _weights(vgg):
    convs = [m for m in vgg.model if isinstance(m, torch.nn.Conv2d)]
    return [(m.weight.detach(), m.bias.detach()) for m in convs]


# ---- every launch on its own input ---------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("wset", V.WEIGHT_SETS)
def test_every_launch_against_its_float64_replay(wset, shape):
    """The 20 forward launches, the seed and the 20 backward launches of one (out, ref) pair, each replayed in float64
    from the GPU's own decoded input (ReLU' from the GPU's saved planes, pools routed by them), and the fold of
    d(out); the loss is the float64 sum over the GPU's own conv5_4 features of out and ref.  Both weight sets of
    vgg_reference: the default init's biases are all 0."""
    bf16, _ = _modes()
    out, ref = _pair(*shape, seed=sum(shape))
    vgg = V.perceptual_model(wset, precision="bf16")
    eng = vgg._vgg_engine(out)
    ws = _weights(vgg)
    dbg = lambda x, k, r=None: eng.debug_vgg_layer(x, k, ref=r, train_mode=bf16).double()
    fwd = [dbg(out, k) for k in range(20)]
    fref = dbg(ref, 19)
    seed = dbg(out, 21, ref)
    bwd = [dbg(out, 22 + k, ref) for k in range(20)]
    assert torch.count_nonzero(bwd[0][:, 3:]) == 0  # 16 normalised channels, 3 real
    bwd[0] = bwd[0][:, :3]
    act0 = vr._bf16(vr._norm_f32(out))  # the pack's planes, as the first launch reads them
    worst = {"forward": 0.0, "backward": 0.0}
    for k in range(20):
        worst["forward"] = max(worst["forward"], vr.check_forward_launch(k, act0, fwd, ws))
        worst["backward"] = max(worst["backward"], vr.check_backward_launch(k, fwd, seed, bwd, ws))
    worst["seed"] = vr.check_seed(seed, fwd[19], fref)
    for kind, v in worst.items():
        _report(f"{kind} {wset} {shape}", v)
    loss, g = eng.perceptual_loss(out, ref, want_grad=True, train_mode=bf16)
    want = vr.loss_from_features(fwd[19], fref)
    assert abs(loss.item() - want) <= 2.0 ** -22 * want, (loss.item(), want)
    R = bwd[0] / vr._std64(out.device)
    vr.rp.check(g, vr.types.SimpleNamespace(R=R, M=R.abs()), FOLD_TAU, "fold of d(out)")


def test_the_first_launch_reads_the_bf16_pack(vgg):
    """The replay of launch 0 from bf16((v - mean) / std) alone: a pack that kept a lo plane (or a launch that read
    one) fails it."""
    bf16, _ = _modes()
    out, _ = _pair(2, 40, 56, seed=3)
    eng = vgg._vgg_engine(out)
    G = eng.debug_vgg_layer(out, 0, train_mode=bf16).double()
    w, b = _weights(vgg)[0]
    ref = vr.fwd_replay(vr._bf16(vr._norm_f32(out)), w, b)
    vr.rp.check(G, ref, vr.acc_tau(vr.fwd_k(0)), "conv1_1 from the pack", planes=True)


# ---- windows -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tile", [16, 32, 48, (48, 32), 128])
def test_windows_match_one_window(vgg, tile):
    bf16, _ = _modes()
    out, ref = _pair(2, 200, 264, seed=11)
    eng = vgg._vgg_engine(out)
    f1 = eng.debug_vgg_layer(out, 20, train_mode=bf16)
    ft = eng.debug_vgg_layer(out, 20, tile=tile, train_mode=bf16)
    assert torch.equal(f1, ft)
    l1, g1 = eng.perceptual_loss(out, ref, want_grad=True, train_mode=bf16)
    lt, gt = eng.perceptual_loss(out, ref, tile=tile, want_grad=True, train_mode=bf16)
    assert abs(lt.item() - l1.item()) <= 1e-6 * l1.item()
    e = _rel(gt, g1)
    _report(f"seam_grad{tile}", e)
    assert e <= SEAM_GRAD_REL, e


# ---- determinism, strides, sizes -----------------------------------------------------------------------------------
def test_deterministic_across_calls_pass_sizes_and_workspace_contents(vgg):
    bf16, _ = _modes()
    out, ref = _pair(2, 160, 200, seed=9)
    eng = vgg._vgg_engine(out)
    base = eng.perceptual_loss(out, ref, tile=48, want_grad=True, train_mode=bf16)
    for mpp in (0, 20_000, 70_000, 8 << 20):
        ws = eng._ws.get("vgg")
        if ws is not None:
            ws.fill_(0xFF)
        got = eng.perceptual_loss(out, ref, tile=48, want_grad=True, max_pass_pixels=mpp, train_mode=bf16)
        assert torch.equal(got[0], base[0]) and torch.equal(got[1], base[1]), mpp


@pytest.mark.parametrize("shape", [(1, 16, 16), (1, 17, 31), (1, 37, 53), (1, 113, 117), (1, 300, 500), (3, 40, 72)])
def test_odd_sizes_and_strided_inputs(vgg, shape):
    bf16, _ = _modes()
    out, ref = _pair(*shape, seed=5)
    eng = vgg._vgg_engine(out)
    l0, g0 = eng.perceptual_loss(out, ref, tile=32, want_grad=True, train_mode=bf16)
    cl = [t.contiguous(memory_format=torch.channels_last) for t in (out, ref)]
    l1, g1 = eng.perceptual_loss(cl[0], cl[1], tile=32, want_grad=True, train_mode=bf16)
    assert torch.equal(l0, l1) and torch.equal(g0, g1)
    assert torch.isfinite(g0).all() and l0.item() > 0


# ---- the mode of a handle ------------------------------------------------------------------------------------------
def test_modes_do_not_leak_between_calls(vgg):
    """A bf16x3 call on a handle switched to bf16 and back is the bits of one on a fresh handle; the bf16 results are
    the same on both handles."""
    bf16, bf16x3 = _modes()
    out, ref = _pair(2, 48, 80, seed=13)
    fresh_vgg = _vgg(precision="bf16x3")
    fresh = fresh_vgg._vgg_engine(out)
    want = fresh.perceptual_loss(out, ref, tile=32, want_grad=True, train_mode=bf16x3)
    eng = vgg._vgg_engine(out)
    b1 = eng.perceptual_loss(out, ref, tile=32, want_grad=True, train_mode=bf16)
    got = eng.perceptual_loss(out, ref, tile=32, want_grad=True, train_mode=bf16x3)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    b2 = fresh.perceptual_loss(out, ref, tile=32, want_grad=True, train_mode=bf16)
    assert torch.equal(b1[0], b2[0]) and torch.equal(b1[1], b2[1])
    assert not torch.equal(b1[1], want[1])  # the two arithmetics differ
    f1 = eng.debug_vgg_layer(out, 5, train_mode=bf16x3)
    assert torch.equal(f1, fresh.debug_vgg_layer(out, 5, train_mode=bf16x3))


# ---- autograd ------------------------------------------------------------------------------------------------------
def test_autograd_returns_the_scaled_gradient_and_leaves_vgg_alone():
    from waternet_b200.training import perceptual_loss
    bf16, bf16x3 = _modes()
    v = _vgg(precision="bf16")
    out, ref = _pair(2, 48, 64, seed=4)
    eng = v._vgg_engine(out)
    lb, gb = eng.perceptual_loss(out, ref, want_grad=True, train_mode=bf16)
    lx, gx = eng.perceptual_loss(out, ref, want_grad=True, train_mode=bf16x3)
    o = out.clone().requires_grad_(True)
    perc = perceptual_loss(v, o, ref)
    (0.05 * perc).backward()
    assert torch.equal(perc.detach(), lb)
    assert torch.allclose(o.grad, 0.05 * gb, rtol=1e-6, atol=0)
    assert all(p.grad is None for p in v.parameters())
    # eval: the bf16 forward alone, the same loss
    with torch.no_grad():
        l2 = perceptual_loss(v, o, ref)
    assert l2.grad_fn is None and torch.equal(l2, lb)
    # a change of precision takes effect at the next call
    v.precision = "bf16x3"
    o.grad = None
    perc = perceptual_loss(v, o, ref)
    perc.backward()
    assert torch.equal(perc.detach(), lx) and torch.equal(o.grad, gx)
    assert not torch.equal(gx, gb)


# ---- buffer bounds in this mode ------------------------------------------------------------------------------------
BOUNDS = [s for s in bb.ROW["perceptual_loss"].specs if s.get("shape") != bb.BIG]


@pytest.fixture(scope="module")
def bounds_eng():
    from waternet_b200.engine import new_engine
    e = new_engine("cuda:0")
    e.pack_vgg_weights(bb.vgg_params())
    yield e


@pytest.mark.parametrize("spec", BOUNDS, ids=[bb.spec_id(s) for s in BOUNDS])
def test_perceptual_loss_stays_inside_its_buffers(bounds_eng, spec):
    """Guards, the exact workspace at the four offsets with different poison (the same bits, no NaN, the Engine
    call's bits), one byte short refused, with the handle in WN_MODE_BF16."""
    bf16, _ = _modes()
    eng, row = bounds_eng, bb.ROW["perceptual_loss"]
    plan = row.build(spec)
    results = []
    for k, off in enumerate(bb.START_OFFSETS):
        eng.set_train_mode(bf16)
        rc, P, ws = _run(eng, row, spec, plan, offset=off, poison=k % 2, ws_fill=(k ^ (k >> 1)) & 1)
        _ok(eng, rc, P, ws, f"offset {off}")
        results.append(_outputs(plan, P))
        del P, ws
    for res in results[1:]:
        for name, t in results[0].items():
            assert torch.equal(t.contiguous().view(-1).view(torch.uint8), res[name].contiguous().view(-1).view(
                torch.uint8)), name
    for name, t in results[0].items():
        assert not bool(torch.isnan(t).any()), name
    T = {b.name: b.data.cuda() for b in plan.bufs if b.role == "in"}
    th, tw = spec["tile"]
    loss, grad = eng.perceptual_loss(T["out"], T["ref"], tile=None if th == 0 else (th, tw),
                                     want_grad=spec.get("grad", True), max_pass_pixels=spec["mpp"], train_mode=bf16)
    assert torch.equal(results[0]["loss"], loss.reshape(1))
    if grad is not None:
        assert torch.equal(results[0]["grad"], grad)
    need = bb.workspace_bytes(eng.lib, row, spec)
    eng.set_train_mode(bf16)
    rc, P, ws = _run(eng, row, spec, plan, ws_bytes=need - 1)
    assert rc == -4, f"one byte short: code {rc}"


# ---- training ------------------------------------------------------------------------------------------------------
def test_training_epochs_track_the_bf16x3_vgg():
    """The 3-epoch loop of test_perceptual_gpu.test_training_epochs_track_the_torch_vgg with the native loss in bf16
    and in bf16x3: every row (train loss, train and validation perceptual loss, validation MSE) within TRAIN_REL."""
    from waternet.net import WaterNet
    from waternet.training_utils import GpuBatchLoader, SyntheticUIEB
    from waternet_b200 import training as T
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ds = SyntheticUIEB(12, 48, 64, seed=2)
    hist = []
    for precision in ("bf16x3", "bf16"):
        torch.manual_seed(0)
        model = WaterNet().cuda().train()
        vgg = T.PerceptualModel(pretrained=False, native=True, precision=precision).cuda().eval()
        opt = torch.optim.Adam(model.parameters(), lr=1e-3)
        sched = torch.optim.lr_scheduler.StepLR(opt, step_size=10000, gamma=0.1)
        rows = []
        for _ in range(3):
            loader = GpuBatchLoader(ds, 4, "cuda:0", augment=False)
            tm = T.train_one_epoch(model, loader, opt, sched, vgg, "cuda")
            vm = T.eval_one_epoch(model, GpuBatchLoader(ds, 4, "cuda:0", augment=False), vgg, "cuda")
            rows.append([tm["loss"], tm["perceptual_loss"], vm["perceptual_loss"], vm["mse"]])
        hist.append(np.array(rows))
    worst = float(np.max(np.abs(hist[1] - hist[0]) / np.abs(hist[0])))
    _report("train_rows", worst)
    print("training rows bf16x3 / bf16", hist, "worst relative difference", worst)
    assert TRAIN_REL <= 0.05
    assert worst <= TRAIN_REL, (worst, hist)
