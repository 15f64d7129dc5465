"""The per-launch backward check of test_backward_layers_gpu.py tells the documented arithmetic from weaker ones.

backward_reference.emulate_* restate the operand formats of the seeds, the data-gradient launches and the weight- and
bias-gradient reductions with exact float64 products, on the saved buffers of forward_reference's bf16x3 emulation.
Their results must pass the committed bars at every launch, on every weight set and input kind (else tau was fitted
to luck); and each fault of backward_reference.FAULTS -- a ReLU' mask read one pixel off, from the wrong half of a bf16
pair, missing, or zeroed at a tile edge, unrotated taps, a dropped correction pass, a missing tile or tap group, a bias
from the hi planes only, a seed without its (1 - cm) factor or ReLU' mask, a first layer without its 1/255 or with it
twice, a refiner reading the next refiner's channels -- must fail the bar of the launch it targets.
"""
import pytest
import torch

import backward_reference as br
import forward_reference as fr

SHAPE = (1, 19, 24)  # one full 16 x 16 tile and partial ones on both axes


@pytest.fixture(scope="module", autouse=True)
def _threads():
    n = torch.get_num_threads()
    torch.set_num_threads(min(8, n))
    yield
    torch.set_num_threads(n)


def _grad(seed):
    return torch.randn(SHAPE[0], 3, *SHAPE[1:], generator=torch.Generator().manual_seed(seed))


def _values(bufs):
    return {k: v.value for k, v in bufs.items()}


def _check_all(sd, stack, grad, bufs, params, which=0, label=""):
    """Every seed, launch and parameter gradient of one emulated backward against its reference."""
    vals = _values(bufs)
    seeds = br.seed_reference(stack, grad, vals.get("cm"), vals.get("refined"), which)
    for name, ref in seeds.items():
        br.check(vals[name], ref, br.TAU["seed"], f"{label} {name}")
    for li in br.DGRAD:
        if li in vals:
            mask = br.DGRAD_MASK[li]
            ref = br.dgrad_reference(sd, li, vals[br.DGRAD_INPUT[li]], vals[mask] if mask else None)
            br.check(vals[li], ref, br.TAU["dgrad"], f"{label} {li}")
    for prefix, (dw, db) in params.items():
        wref, bref = br.param_reference(prefix, vals)
        # the emulation sums exactly: the tightest weight-gradient bar, that of the shortest partial sum
        br.check(dw, wref, br.wgrad_tau(0), f"{label} {prefix}.weight")
        br.check(db, bref, br.TAU["bias"], f"{label} {prefix}.bias")


def _fold(stack, vals, which=0):
    """extract_input_grads_kernel's fp32 sums ((hi_a + lo_a) + hi_b) + lo_b, or its copy of one buffer."""
    if stack == "all":
        a, b = vals["kD1"], vals["kDR1"]
        return [a[:, 3 * t:3 * t + 3] + b[:, 3 * t:3 * t + 3] for t in range(4)]
    return [r.R for r in br.fold_reference(stack, vals.get("kD1"), vals.get("kDR1"), which)]


@pytest.mark.parametrize("weights", fr.WEIGHT_SETS)
def test_emulated_arithmetic_passes_the_bar(weights):
    """Every seed, launch and parameter gradient of the emulated backward of each stack, for every input kind."""
    sd = fr.weight_set(weights, 1)
    for i, kind in enumerate(fr.INPUT_KINDS):
        ins = fr.make_inputs(kind, *SHAPE, 60 + i)
        fwd = br.emulate_forward(sd, ins)
        for stack, which in (("all", 0), ("cmg", 0), ("refiner", i % 3)):
            grad = _grad(70 + i)
            bufs, params = br.emulate_backward(sd, stack, grad, fwd, which)
            _check_all(sd, stack, grad, bufs, params, which, f"{weights} {kind} {stack}")


def test_emulated_fold_passes_the_bar():
    """The fp32 fold of the two first-layer launches is within TAU["fold"] of their float64 sum."""
    sd = fr.weight_set("stress", 1)
    ins = fr.make_inputs("floats", *SHAPE, 80)
    bufs, _ = br.emulate_backward(sd, "all", _grad(81), br.emulate_forward(sd, ins))
    vals = _values(bufs)
    for t, ref in enumerate(br.fold_reference("all", vals["kD1"], vals["kDR1"])):
        a, b = bufs["kD1"], bufs["kDR1"]
        f32 = lambda x: x.float().double()
        got = f32(f32(f32(a.hi + a.lo) + b.hi) + b.lo)[:, 3 * t:3 * t + 3]
        br.check(got, ref, br.TAU["fold"], f"fold {t}")


# (fault, where): the seed, launch or convolution that computes wrongly
REJECTED = [
    ("mask_right", "kD5"), ("mask_right", "kDR3"),
    ("mask_down", "kD3"),
    ("mask_pair_swap", "kD7"), ("mask_pair_swap", "kDR2"),
    ("no_mask", "kD8"), ("no_mask", "kDR2"),
    ("mask_tile_row", "kD2"),
    ("mask_tile_column", "kDR3"),
    ("unrotated_taps", "kD6"), ("unrotated_taps", "kD1"),
    ("drop_g_lo", "kD4"), ("drop_g_lo", "kDR1"),
    ("drop_a_lo", "cmg.conv3"), ("drop_a_lo", "cmg.conv1"),
    ("missing_tile", "cmg.conv5"), ("missing_tile", "gc_refiner.conv2"),
    ("zero_tap_group", "cmg.conv5"),
    ("bias_hi_only", "cmg.conv2"), ("bias_hi_only", "wb_refiner.conv3"),
    ("seed_no_one_minus_cm", "g8"),
    ("seed_no_refined_mask", "gr3"),
    ("first_layer_no_255", "cmg.conv1"),
    ("first_layer_255_twice", "wb_refiner.conv1"),
    ("refiner_next_channels", "ce_refiner.conv1"),
]


def test_every_fault_is_listed():
    assert {f for f, _ in REJECTED} == set(br.FAULTS)


@pytest.mark.parametrize("fault,where", REJECTED)
def test_check_rejects_fault(fault, where):
    sd = fr.weight_set("stress", 1)
    ins = fr.make_inputs("floats", *SHAPE, 40)
    grad = _grad(41)
    fwd = br.emulate_forward(sd, ins)
    bufs, params = br.emulate_backward(sd, "all", grad, fwd, fault=fault, fault_at=where)
    vals = _values(bufs)
    if where in ("g8", "gr3"):
        ref = br.seed_reference("all", grad, vals["cm"], vals["refined"])[where]
        got, tau = vals[where], br.TAU["seed"]
    elif where in br.DGRAD:
        mask = br.DGRAD_MASK[where]
        ref = br.dgrad_reference(sd, where, vals[br.DGRAD_INPUT[where]], vals[mask] if mask else None)
        got, tau = vals[where], br.TAU["dgrad"]
    else:
        wref, bref = br.param_reference(where, vals)
        bias = fault == "bias_hi_only"
        ref, got = (bref, params[where][1]) if bias else (wref, params[where][0])
        # the loosest weight-gradient bar the GPU suite uses, that of the largest partial sum (1 x 385 x 577)
        li = br.WGRAD_SPECS[where][0]
        tau = br.TAU["bias"] if bias else br.wgrad_tau(br.wgrad_pixels(li, 1, 385, 577, 132))
        where += ".bias" if bias else ".weight"
    with pytest.raises(AssertionError):
        br.check(got, ref, tau, f"{fault}: {where}")
