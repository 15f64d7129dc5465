"""The float64 gradient reference and its element-wise check (tests/grad_reference.py), on the CPU: the check
passes gradients within a 1e-5 relative perturbation of the reference and rejects each of the localized errors
a backward kernel could make -- the errors a whole-tensor norm would hide."""
import pytest
import torch

from grad_reference import (INPUT_NAMES, PARAM_NAMES, RELU_LAYERS, TAU, assert_grad_close, assert_relus_cannot_flip,
                            dead_channels, gated_state_dict, reference, smooth_state_dict)

N, H, W = 2, 24, 40


@pytest.fixture(scope="module", params=["smooth", "gated"])
def case(request):
    sd = (smooth_state_dict if request.param == "smooth" else gated_state_dict)(11)
    gen = torch.Generator().manual_seed(12)
    ins = [torch.rand(N, 3, H, W, generator=gen) for _ in range(4)]
    grad = torch.randn(N, 3, H, W, generator=gen)
    ref = reference(sd, ins, grad)
    ref.sd, ref.ins, ref.seed, ref.kind = sd, ins, grad, request.param
    return ref


def _tensors(ref):
    """(name, R, M) for the 34 parameter gradients and the 4 input-image gradients."""
    return [(k, ref.grads[k], ref.M[k]) for k in PARAM_NAMES] + \
           [(n, r, m) for n, r, m in zip(INPUT_NAMES, ref.input_grads, ref.M_inputs)]


def _fails(G, R, M, name):
    with pytest.raises(AssertionError):
        assert_grad_close(G, R, M, TAU, name)


def test_premise_and_magnitude_bound(case):
    assert_relus_cannot_flip(case.z)
    for name, r, m in _tensors(case):
        assert (m >= 0).all() and (r.abs() <= m * (1 + 1e-12)).all(), name   # |R| <= M: M bounds the terms
        assert (m > 0).any(), name
    if case.kind == "gated":
        for layer in RELU_LAYERS:
            dead = dead_channels(layer)
            assert dead and (case.z[layer][:, dead] < 0).all() and (case.z[layer][:, [
                c for c in range(case.z[layer].shape[1]) if c not in dead]] > 0).all(), layer
            assert (case.grads[layer + ".weight"][dead] == 0).all() and (case.grads[layer + ".bias"][dead] == 0).all()
            assert (case.M[layer + ".weight"][dead] == 0).all()


def test_reference_matches_mse_seed(case):
    """The target form of the seed is mse_loss's gradient."""
    target = torch.rand(N, 3, H, W, generator=torch.Generator().manual_seed(13))
    a = reference(case.sd, case.ins, target=target, magnitude=False)
    b = reference(case.sd, case.ins, grad=2 * (a.out - target.double()) / a.out.numel(), magnitude=False)
    for k in PARAM_NAMES:
        assert (a.grads[k] - b.grads[k]).abs().max() <= 1e-12 * a.grads[k].abs().max(), k


def test_small_relative_noise_passes(case):
    gen = torch.Generator().manual_seed(14)
    for name, r, m in _tensors(case):
        noise = torch.rand(r.shape, generator=gen, dtype=torch.float64) * 2 - 1
        assert_grad_close(r * (1 + 1e-5 * noise), r, m, TAU, name)


def test_tap_shifted_by_one_fails(case):
    for name in ("cmg.conv1.weight", "cmg.conv5.weight", "cmg.conv8.weight", "ce_refiner.conv2.weight"):
        r, m = case.grads[name], case.M[name]
        g = r.clone()
        g[:, :, 1, 1] = r[:, :, 1, 2]       # one tap reads its right-hand neighbour
        _fails(g, r, m, name)


def test_two_output_channels_swapped_fails(case):
    for name in ("cmg.conv3.weight", "cmg.conv4.bias", "gc_refiner.conv1.weight", "wb_refiner.conv3.weight"):
        r, m = case.grads[name], case.M[name]
        a, b = (0, 2) if r.shape[0] == 3 else (5, 9)
        g = r.clone()
        g[[a, b]] = r[[b, a]]
        _fails(g, r, m, name)


def test_one_dgrad_tile_dropped_fails(case):
    for i, name in enumerate(INPUT_NAMES):
        r, m = case.input_grads[i], case.M_inputs[i]
        g = r.clone()
        g[1, :, 8:16, 16:32] = 0            # one 8 x 16 tile of the second image
        _fails(g, r, m, name)


def test_one_edge_row_zeroed_fails(case):
    for i, name in enumerate(INPUT_NAMES):
        r, m = case.input_grads[i], case.M_inputs[i]
        for rows in (slice(0, 1), slice(H - 1, H)):
            g = r.clone()
            g[0, :, rows] = 0
            _fails(g, r, m, name)
        g = r.clone()
        g[0, :, :, W - 1] = 0               # and the last column
        _fails(g, r, m, name)


def test_one_image_dropped_from_parameter_gradients_fails(case):
    """Gradients of the first image alone: every one of the 34 parameter gradients must be rejected."""
    first = reference(case.sd, [t[:1] for t in case.ins], grad=case.seed[:1], magnitude=False)
    for name in PARAM_NAMES:
        r, m = case.grads[name], case.M[name]
        _fails(first.grads[name], r, m, name)
