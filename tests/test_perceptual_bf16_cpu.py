"""The single-pass bf16 VGG arithmetic of the native perceptual loss (PerceptualModel(precision="bf16"),
wn_set_train_mode(WN_MODE_BF16) on the VGG handle) without a GPU: its float64 replay bars, and the Python surface.

emulate_forward / emulate_backward restate the kernels of that mode with exact float64 products on small images:
the packed image stored as bf16((v - mean) / std) with lo = 0; every convolution ONE bf16 product a_hi x w_hi (weights
rounded to bf16 with round to nearest even), fp32 results, stored as bf16 with lo = 0; pools that choose on hi (the
first maximum in row-major order); the seed bf16 with lo = 0.  Each launch must pass its replay bar, acc_tau(K) M +
2^-8 |R| (K = cinpad x 9 for a forward launch, the forward cout x 9 for a data gradient), replayed from the emulation's
own decoded input, and the exact-arithmetic bar (unrounded weights, 2^-8 M more).  Each fault of FAULT_CASES must fail
the bar of the launch it targets.

The replay helpers (fwd_replay, dgrad_replay, seed_replay, pack_replay) are shared with test_perceptual_bf16_gpu.py,
which replays every launch of the GPU from its own decoded input in the same way.
"""
import argparse
import json
import pickle
import types

import pytest
import torch
import torch.nn.functional as F

import bf16_replay as rp
import vgg_reference as V
from bf16_replay import _bf16, acc_tau
from vgg_reference import CONVS, MEAN, STD, STEPS

ROUND = 2.0 ** -8
PACK_TAU = 2.0 ** -22  # (v - mean) / std: two fp32 operations, then the bf16 store (F)

def fwd_k(conv):
    """Products per output element of forward convolution ``conv``: cinpad x 9 (the first one reads 16 channels)."""
    return (16 if conv == 0 else CONVS[conv][0]) * 9


def dgrad_k(conv):
    """Products per output element of the data gradient of convolution ``conv``: the forward cout x 9."""
    return CONVS[conv][1] * 9


def _f32(t):
    return t.float().double()


def _hilo(v):
    """v stored as bf16x3 planes (hi + lo): what a store that does not zero lo leaves."""
    h = _bf16(v)
    return h + _bf16(v - h)


def _norm_f32(x):
    """(v - mean) / std as vgg_pack_kernel evaluates it: fp32 subtract, fp32 divide."""
    mean = torch.tensor(MEAN, dtype=torch.float32).view(1, 3, 1, 1).to(x.device)
    std = torch.tensor(STD, dtype=torch.float32).view(1, 3, 1, 1).to(x.device)
    return ((x.float() - mean) / std).double()


def _std64(device):
    return torch.tensor(STD, dtype=torch.float32).double().view(1, 3, 1, 1).to(device)


# ------------------------------------------------------------------ replays (float64, from a launch's decoded input)
def pack_replay(x):
    R = _norm_f32(x)
    return types.SimpleNamespace(R=R, M=R.abs(), F=ROUND * R.abs())


def fwd_replay(a, w, b, rounded=True):
    """R, M, F of a forward convolution (+ bias, ReLU, bf16 store) from its decoded input ``a``: the kernel reads the
    hi planes, so ``a`` is rounded to bf16 too (a no-op unless a lo plane was left in)."""
    a = _bf16(a.double())
    w = w.double().to(a.device)
    wr = _bf16(w) if rounded else _f32(w)
    b = b.double().to(a.device)
    R = F.relu(F.conv2d(a, wr, b, padding=1))
    M = F.conv2d(a.abs(), wr.abs(), b.abs(), padding=1)
    return types.SimpleNamespace(R=R, M=M, F=ROUND * R)


def dgrad_replay(g, w, mask, rounded=True):
    """R, M, F of a data-gradient launch from its decoded input gradient ``g`` and the saved forward output whose
    zeros gate it (None: the normalised image, no ReLU in front)."""
    g = _bf16(g.double())
    w = w.double().to(g.device)
    wr = _bf16(w) if rounded else _f32(w)
    R = F.conv_transpose2d(g, wr, padding=1)
    M = F.conv_transpose2d(g.abs(), wr.abs(), padding=1)
    if mask is not None:
        on = (mask.double() > 0).double()
        R, M = R * on, M * on
    return types.SimpleNamespace(R=R, M=M, F=ROUND * R.abs())


def seed_replay(fo, fr):
    """The seed d(loss)/d(conv5_4 before its ReLU) from the decoded conv5_4 features of out and ref."""
    fo, fr = fo.double(), fr.double()
    R = 2.0 * 255.0 ** 2 / fo.numel() * (fo - fr) * (fo > 0).double()
    return types.SimpleNamespace(R=R, M=R.abs(), F=ROUND * R.abs())


def pool_replay(a):
    return F.max_pool2d(a.double(), 2, 2)


def pool_bwd_replay(g, saved):
    _, idx = F.max_pool2d(saved.double(), 2, 2, return_indices=True)
    return F.max_unpool2d(g.double(), idx, 2, 2, output_size=saved.shape[-2:])


def pool_bwd_last(g, saved):
    """A pool backward that routes a tie to the LAST maximum of its window: the first one of the window turned
    around (both axes flipped on the even part, the floored edge 0)."""
    h, w = saved.shape[-2] // 2 * 2, saved.shape[-1] // 2 * 2
    _, idx = F.max_pool2d(saved[..., :h, :w].double().flip(-2, -1), 2, 2, return_indices=True)
    r = F.max_unpool2d(g.double().flip(-2, -1), idx, 2, 2, output_size=(h, w)).flip(-2, -1)
    return F.pad(r, (0, saved.shape[-1] - w, 0, saved.shape[-2] - h))


def loss_from_features(fo, fr):
    return (torch.square(255.0 * (fo.double() - fr.double()))).sum().item() / fo.numel()


# ------------------------------------------------------------------ emulation of the kernels' arithmetic
def vgg_weights(seed):
    """Seeded weights of the 16 convolutions ((cout, cin, 3, 3) and (cout,), fp32), He-scaled, with nonzero biases."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for cin, cout in CONVS:
        w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (9 * cin)) ** 0.5
        b = 0.05 * torch.randn(cout, generator=g)
        out.append((w, b))
    return out


def image(n, h, w, seed):
    return torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(seed))


def _bias(ws, conv, fault):
    """The biases forward convolution ``conv`` adds: its own, or those of a fault -- "bias_group0" (every column group
    of 128 channels reads group 0's), "bias_next" (the next convolution's), "no_bias"."""
    b = ws[conv][1].double()
    if fault == "bias_group0":
        return b[torch.arange(b.numel()) % 128]
    if fault == "bias_next":
        return ws[conv + 1][1].double()
    return torch.zeros_like(b) if fault == "no_bias" else b


def emulate_forward(x, ws, fault=None, at=None):
    """(act0, the decoded outputs of the 20 forward launches).  ``at``: "pack" or a launch index."""
    v = _norm_f32(x)
    act0 = _hilo(v) if (fault, at) == ("lo_not_zeroed", "pack") else _bf16(v)
    outs, src = [], act0
    for k, (conv, _, _) in enumerate(STEPS):
        if conv < 0:  # the first maximum of hi (lo = 0) in row-major order, bits copied
            outs.append(pool_replay(src))
            src = outs[-1]
            continue
        w, b = ws[conv]
        w = w.double()
        w_hi = _bf16(w)
        a = src if (fault, at) == ("a_lo_pass", k) else _bf16(src)
        z = F.conv2d(a, w_hi, padding=1)
        if (fault, at) == ("w_lo_pass", k):
            z = z + F.conv2d(a, _bf16(w - w_hi), padding=1)
        b = _bias(ws, conv, fault if at == k else None)
        val = F.relu(_f32(_f32(z) + b.view(1, -1, 1, 1)))
        # an a_lo pass reads the lo plane its producer did not zero
        keep_lo = (fault, at) in (("lo_not_zeroed", k), ("a_lo_pass", k + 1))
        outs.append(_hilo(val) if keep_lo else _bf16(val))
        src = outs[-1]
    return act0, outs


def emulate_seed(fo, fr, fault=None):
    """(the seed planes, the loss) of vgg_seed_kernel: fp32 differences, float64 loss partials."""
    scale = float(torch.tensor(2.0 * 255.0 ** 2 / fo.numel(), dtype=torch.float32))
    d = _f32(fo - fr)
    s = torch.where(fo > 0, _f32(scale * d), torch.zeros_like(d))
    if fault == "seed_fp32":
        seed = s
    elif fault == "lo_not_zeroed":
        seed = _hilo(s)
    else:
        seed = _bf16(s)
    return seed, loss_from_features(fo, fr)


def emulate_backward(fwd, seed, ws, fault=None, at=None):
    """The decoded outputs of the 20 backward launches, bwd[k] = d(loss)/d(input of forward launch k) (k = 0: the 3
    normalised channels), and d(out) as vgg_fold_kernel forms it (fp32, one window).  ``at``: a launch index."""
    bwd = [None] * len(STEPS)
    g = seed
    for k in range(len(STEPS) - 1, -1, -1):
        conv = STEPS[k][0]
        if conv < 0:
            bwd[k] = (pool_bwd_last if (fault, at) == ("ties_last", k) else pool_bwd_replay)(g, fwd[k - 1])
            g = bwd[k]
            continue
        w = ws[conv][0].double()
        w_hi = _bf16(w)
        gi = g if (fault, at) == ("a_lo_pass", k) else _bf16(g)
        z = F.conv_transpose2d(gi, w_hi, padding=1)
        if (fault, at) == ("w_lo_pass", k):
            z = z + F.conv_transpose2d(gi, _bf16(w - w_hi), padding=1)
        z = _f32(z)
        if k:
            mask = fwd[k - 2] if (fault, at) == ("wrong_mask", k) else fwd[k - 1]
            z = z * (mask > 0).double()
        keep_lo = (fault, at) in (("lo_not_zeroed", k), ("a_lo_pass", k - 1))
        bwd[k] = _hilo(z) if keep_lo else _bf16(z)
        g = bwd[k]
    dout = _f32(bwd[0] / _std64(bwd[0].device))
    return bwd, dout


# ------------------------------------------------------------------ the bars
def check_forward_launch(k, act0, fwd, ws, exact=False):
    """Forward launch k against its replay from its own decoded input; returns the worst excess over F, in units of
    M (0 for a pool, which must be exact)."""
    src = act0 if k == 0 else fwd[k - 1]
    conv = STEPS[k][0]
    if conv < 0:
        assert torch.equal(fwd[k], pool_replay(src)), f"pool {k} is not exact"
        return 0.0
    w, b = ws[conv]
    a = src[:, :3] if k == 0 else src
    ref = fwd_replay(a, w, b, rounded=not exact)
    tau = acc_tau(fwd_k(conv))
    rp.check(fwd[k], ref, rp.exact_bar(tau) if exact else tau, f"forward launch {k}", planes=True)
    return rp.excess(fwd[k], ref)


def check_backward_launch(k, fwd, seed, bwd, ws, exact=False):
    """Backward launch k (the data gradient of forward launch k, or a pool's routing) against its replay from its own
    decoded input gradient and the saved forward output that gates it."""
    gin = seed if k == len(STEPS) - 1 else bwd[k + 1]
    conv = STEPS[k][0]
    if conv < 0:
        assert torch.equal(bwd[k], pool_bwd_replay(gin, fwd[k - 1])), f"pool backward {k} is not exact"
        return 0.0
    ref = dgrad_replay(gin, ws[conv][0], fwd[k - 1] if k else None, rounded=not exact)
    tau = acc_tau(dgrad_k(conv))
    rp.check(bwd[k], ref, rp.exact_bar(tau) if exact else tau, f"backward launch {k}", planes=True)
    return rp.excess(bwd[k], ref)


def check_seed(seed, fo, fr):
    ref = seed_replay(fo, fr)
    rp.check(seed, ref, rp.SEED_TAU, "seed", planes=True)
    return rp.excess(seed, ref)


def check_pack(act0, x):
    rp.check(act0, pack_replay(x), PACK_TAU, "pack", planes=True)


SHAPES = ((1, 32, 48), (2, 17, 40))


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(8, n))
    yield
    torch.set_num_threads(n)


@pytest.fixture(scope="module")
def ws():
    return vgg_weights(5)


def _run(ws, shape, fault=None, at=None, kind=None):
    if kind is None:
        out, ref = image(*shape, seed=sum(shape)), image(*shape, seed=sum(shape) + 1)
    else:
        out, ref = V.pair(kind, *shape, seed=sum(shape))
    act0, fwd = emulate_forward(out, ws, fault, at)
    _, fref = emulate_forward(ref, ws)
    seed, loss = emulate_seed(fwd[-1], fref[-1], fault if at == "seed" else None)
    bwd, dout = emulate_backward(fwd, seed, ws, fault, at)
    return types.SimpleNamespace(x=out, act0=act0, fwd=fwd, fref=fref, seed=seed, loss=loss, bwd=bwd, dout=dout)


@pytest.mark.parametrize("shape", SHAPES)
def test_emulation_passes_the_replay_bars(ws, shape):
    e = _run(ws, shape)
    check_pack(e.act0, e.x)
    for k in range(len(STEPS)):
        check_forward_launch(k, e.act0, e.fwd, ws)
    check_seed(e.seed, e.fwd[-1], e.fref[-1])
    for k in range(len(STEPS)):
        check_backward_launch(k, e.fwd, e.seed, e.bwd, ws)
    assert torch.count_nonzero(e.bwd[0][:, :3]) > 0
    # the loss from the decoded features, d(out) one fp32 division from the 3 normalised channels
    assert e.loss == loss_from_features(e.fwd[-1], e.fref[-1]) and e.loss > 0
    R = e.bwd[0] / _std64(e.bwd[0].device)
    assert (e.dout - R).abs().max() <= 2.0 ** -24 * R.abs().max()


@pytest.mark.parametrize("shape", SHAPES)
def test_emulation_passes_the_exact_arithmetic_bars(ws, shape):
    """Against the unrounded fp32 weights every convolution stays within 2^-8 M + its accumulation bar."""
    e = _run(ws, shape)
    for k in range(len(STEPS)):
        check_forward_launch(k, e.act0, e.fwd, ws, exact=True)
        check_backward_launch(k, e.fwd, e.seed, e.bwd, ws, exact=True)


def test_bf16x3_results_fail_the_replay_bars(ws):
    """The bars tell the arithmetics apart: a launch whose result kept the bf16x3 lo plane fails."""
    e = _run(ws, SHAPES[0], "lo_not_zeroed", 1)
    with pytest.raises(AssertionError):
        check_forward_launch(1, e.act0, e.fwd, ws)


# (fault, where it is injected, which bar must fail): forward launch k, backward launch k, the pack or the seed
FAULT_CASES = [
    ("w_lo_pass", 4, "forward"), ("w_lo_pass", 12, "backward"),
    ("a_lo_pass", 7, "forward"), ("a_lo_pass", 13, "backward"),
    ("lo_not_zeroed", "pack", "pack"), ("lo_not_zeroed", 9, "forward"), ("lo_not_zeroed", 16, "backward"),
    ("lo_not_zeroed", "seed", "seed"), ("seed_fp32", "seed", "seed"),
    ("wrong_mask", 8, "backward"), ("wrong_mask", 18, "backward"),
]


@pytest.mark.parametrize("fault,at,kind", FAULT_CASES)
def test_each_fault_fails_its_launch(ws, fault, at, kind):
    e = _run(ws, SHAPES[0], fault, at)
    with pytest.raises(AssertionError):
        if kind == "pack":
            check_pack(e.act0, e.x)
        elif kind == "seed":
            check_seed(e.seed, e.fwd[-1], e.fref[-1])
        elif kind == "forward":
            check_forward_launch(at, e.act0, e.fwd, ws)
        else:
            check_backward_launch(at, e.fwd, e.seed, e.bwd, ws)


# the weights and images of vgg_reference: nonzero biases at each layer's spread, flat patches whose pools meet ties;
# (fault, launch, which bar must fail).  Launch 6 is conv3_1 (2 column groups), 11 conv4_1 (4), 12 conv4_2.
BIAS_FAULT_CASES = [
    ("bias_group0", 6, "forward"), ("bias_group0", 11, "forward"), ("bias_next", 12, "forward"),
    ("no_bias", 1, "forward"), ("no_bias", 17, "forward"),
    ("ties_last", 2, "backward"), ("ties_last", 5, "backward"),
]


@pytest.fixture(scope="module")
def biased():
    return V.weights("biased")


def test_emulation_on_biased_weights_and_flat_images_passes_the_replay_bars(biased):
    e = _run(biased, SHAPES[0], kind="flat")
    for k in range(len(STEPS)):
        check_forward_launch(k, e.act0, e.fwd, biased)
        check_backward_launch(k, e.fwd, e.seed, e.bwd, biased)
    # the tie fault below has something to route: tied positive maxima that receive a gradient, at both pools
    for k in (2, 5):
        saved, g = e.fwd[k - 1], e.bwd[k + 1]
        assert not torch.equal(pool_bwd_replay(g, saved), pool_bwd_last(g, saved)), k


@pytest.mark.parametrize("fault,at,kind", BIAS_FAULT_CASES)
def test_each_bias_or_tie_fault_fails_its_launch(biased, fault, at, kind):
    e = _run(biased, SHAPES[0], fault, at, kind="flat")
    with pytest.raises(AssertionError):
        if kind == "forward":
            check_forward_launch(at, e.act0, e.fwd, biased)
        else:
            check_backward_launch(at, e.fwd, e.seed, e.bwd, biased)


# ------------------------------------------------------------------ the Python surface
def test_precision_attribute_is_validated():
    from waternet_b200 import _lib
    from waternet_b200.training import PerceptualModel
    m = PerceptualModel(pretrained=False, native=True)
    assert m.precision == "bf16x3" and m._train_mode() == _lib.MODE_BF16X3
    m = PerceptualModel(pretrained=False, native=True, precision="bf16")
    assert m._train_mode() == _lib.MODE_BF16
    m.precision = "fp8"
    with pytest.raises(ValueError, match="unknown precision"):
        m._train_mode()
    with pytest.raises(ValueError, match="unknown precision"):
        PerceptualModel(pretrained=False, native=True, precision="tf32")
    with pytest.raises(ValueError, match="needs native=True"):
        PerceptualModel(pretrained=False, precision="bf16")
    assert PerceptualModel(pretrained=False).precision == "bf16x3"  # the torch expression keeps the default


def test_a_module_pickled_without_the_attribute_loads_as_bf16x3():
    from waternet_b200 import _lib
    from waternet_b200.training import PerceptualModel
    m = PerceptualModel(pretrained=False, native=True)
    del m.precision  # the state of a module pickled before the attribute existed
    assert "precision" not in m.__dict__
    back = pickle.loads(pickle.dumps(m))
    assert back.precision == "bf16x3" and back._train_mode() == _lib.MODE_BF16X3


def _args(*argv):
    from waternet_b200 import training as T
    ap = argparse.ArgumentParser()
    T.add_perceptual_args(ap)
    return ap.parse_args(list(argv))


@pytest.mark.parametrize("argv", [("--perceptual-precision", "bf16"), ("--perceptual-precision", "bf16x3"),
                                  ("--perceptual", "torch", "--perceptual-precision", "bf16")])
def test_perceptual_precision_needs_native(argv):
    from waternet_b200 import training as T
    with pytest.raises(SystemExit, match="--perceptual-precision needs --perceptual native"):
        T.perceptual_model(_args(*argv))


def test_perceptual_precision_choices():
    with pytest.raises(SystemExit):
        _args("--perceptual", "native", "--perceptual-precision", "fp16")
    assert _args().perceptual_precision is None


def test_config_json_carries_the_perceptual_precision(tmp_path):
    from waternet_b200 import training as T
    for argv, want in ((("--perceptual", "native", "--perceptual-precision", "bf16"), "bf16"), ((), "bf16x3")):
        args = _args(*argv)
        T.save_metrics(tmp_path, None, None, {"epochs": 1, **T.perceptual_config(args)})
        got = json.loads((tmp_path / "config.json").read_text())
        assert got["perceptual_precision"] == want
        assert got["perceptual"] == args.perceptual
