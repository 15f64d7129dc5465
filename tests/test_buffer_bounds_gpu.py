"""Where every C-ABI call writes and what it reads, on the GPU.

Each buffer of a call sits in a guarded arena of its own (tests/buffer_bounds.py): a store past a workspace, an
output or a peer mirror lands in a 1 MiB guard and fails here with its offsets, a write into an input shows as a
changed input, an output element left unwritten or a workspace byte read before it is written shows as a difference
between two runs with different poison, and a read outside an input view (a halo pixel, a reflect or clamp that is
off by one) pulls NaN from the poisoned parent into the result.
"""
import re

import numpy as np
import pytest
import torch

import buffer_bounds as bb

pytestmark = pytest.mark.gpu

CASES = [(r, s) for r in bb.ROWS for s in r.specs]
CASE_IDS = [f"{r.name}-{bb.spec_id(s)}" for r, s in CASES]
WS_CASES = [(r, s) for r, s in CASES if r.ws]
WS_IDS = [f"{r.name}-{bb.spec_id(s)}" for r, s in WS_CASES]
NCHW_ROWS = {r.name for r in bb.ROWS if any(b.nchw for b in r.build(r.specs[0]).bufs)}
STRIDED = [(r, s) for r, s in CASES if r.name in NCHW_ROWS and s.get("shape") != bb.BIG]
# the same with 8-bit level inputs, whose first-layer exact-levels decision scans every input element
STRIDED += [(r, dict(s, levels=True)) for r, s in STRIDED if r.name != "perceptual_loss"]
STRIDED_IDS = [f"{r.name}-{bb.spec_id(s)}" for r, s in STRIDED]
RAGGED = [(r, s) for r, s in CASES if len(s.get("sizes", ())) > 1]
RAGGED_IDS = [f"{r.name}-{bb.spec_id(s)}" for r, s in RAGGED]


@pytest.fixture(scope="module")
def eng():
    from waternet_b200.engine import new_engine
    e = new_engine("cuda:0")
    e.pack_weights(bb.waternet_params())
    e.pack_vgg_weights(bb.vgg_params())
    torch.cuda.reset_peak_memory_stats()
    yield e
    torch.cuda.synchronize()
    print(f"\nbuffer bounds: peak device memory {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB")


def _bits(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _assert_same_bits(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        x, y = _bits(a[k]), _bits(b[k])
        assert x.numel() == y.numel(), f"{what}: {k} has another size"
        diff = torch.nonzero(x != y).flatten()
        assert diff.numel() == 0, f"{what}: {k} differs in {diff.numel()} bytes, first at byte {int(diff[0])}"


def _run(eng, row, spec, plan, offset=0, poison=0, ws_fill=0, layout="contiguous", packed=False, ws_bytes=None,
         gap=None):
    """One call with every buffer in its own arena.  Returns (rc, placed buffers, workspace arena or None)."""
    P = bb.place(plan.bufs, offset, poison, layout, packed, gap=gap)
    ws = None
    nb = 0
    if row.ws:
        nb = bb.workspace_bytes(eng.lib, row, spec) if ws_bytes is None else ws_bytes
        ws = bb.Arena("workspace", nb, offset, seed=77).poison("u8", ws_fill)
    torch.cuda.synchronize()
    with torch.cuda.device(eng.device):
        rc = plan.issue(P, ws.ptr if ws else None, nb, bb._stream(), eng)
    torch.cuda.synchronize()
    return rc, P, ws


def _error(eng):
    msg = eng.lib.wn_last_error()
    return msg.decode() if msg else ""


def _outputs(plan, P):
    return {b.name: P.views[b.name].clone() for b in plan.bufs if b.role == "out"}


def _ok(eng, rc, P, ws, what):
    assert rc == 0, f"{what}: code {rc}: {_error(eng)}"
    bb.check(P.arenas + ([ws] if ws else []))


def _inputs(plan):
    return {b.name: b.data.cuda() for b in plan.bufs if b.role == "in"}


def _release(eng, spec):
    if spec.get("shape") == bb.BIG or any(h * w > 1 << 20 for h, w in spec.get("sizes", [])):
        eng.release_workspaces()
        torch.cuda.empty_cache()


# -------------------------------------------------------------------- 1, 2, 4: exact workspace, full writes, no reads
@pytest.mark.parametrize("row,spec", CASES, ids=CASE_IDS)
def test_exact_workspace_full_writes_and_no_uninitialised_reads(eng, row, spec):
    """The call at the four start offsets (mod 1024) with a workspace of exactly wn_*_workspace_bytes: every guard
    holds and every input is unchanged.  The outputs start as NaN, then -0.0 / 1e30, and the workspace as 0x00, then
    0xFF (both combinations): the results are the same bits, with no NaN, and equal the Engine call on plain
    contiguous tensors.  A pair (forward, backward) poisons its workspace before the forward only."""
    plan = row.build(spec)
    results = []
    for k, off in enumerate(bb.START_OFFSETS):
        rc, P, ws = _run(eng, row, spec, plan, offset=off, poison=k % 2, ws_fill=(k ^ (k >> 1)) & 1)
        _ok(eng, rc, P, ws, f"offset {off}")
        results.append(_outputs(plan, P))
        del P, ws
    _release(eng, spec)
    for k in range(1, 4):
        _assert_same_bits(results[0], results[k], f"offset {bb.START_OFFSETS[k]} against offset 0")
    for name, t in results[0].items():
        if t.dtype == torch.float32:
            assert not bool(torch.isnan(t).any()), f"{name} holds NaN: an element was not written or read poison"
    if plan.engine is not None:
        want = plan.engine(eng, _inputs(plan))
        assert want and set(want) <= set(results[0])
        _assert_same_bits({k: results[0][k] for k in want}, want, "the Engine call")
        del want
    elif row.name in ("pack_weights", "vgg_pack_weights"):
        _check_packed_weights_act_like_the_engines(eng, row)
    _release(eng, spec)


def _check_packed_weights_act_like_the_engines(eng, row):
    """After a pack from guarded arenas the handle computes what it computes after Engine.pack_weights."""
    torch.manual_seed(0)
    if row.name == "pack_weights":
        ins = [torch.rand(1, 3, 25, 17, device="cuda") for _ in range(4)]
        got = eng.forward(*ins, mode=bb.DEFAULT).clone()
        eng.pack_weights(bb.waternet_params())
        want = eng.forward(*ins, mode=bb.DEFAULT)
    else:
        a, b = torch.rand(1, 3, 17, 31, device="cuda"), torch.rand(1, 3, 17, 31, device="cuda")
        got = eng.perceptual_loss(a, b, want_grad=True)[1].clone()
        eng.pack_vgg_weights(bb.vgg_params())
        want = eng.perceptual_loss(a, b, want_grad=True)[1]
    assert torch.equal(_bits(got), _bits(want))


# -------------------------------------------------------------------- 3: strided inputs inside a poisoned parent
@pytest.mark.parametrize("row,spec", STRIDED, ids=STRIDED_IDS)
def test_strided_inputs_read_nothing_outside_the_view(eng, row, spec):
    """fp32 (N,3,H,W) inputs as a slice at an offset, channels_last, and a padded-row view (row stride W + 5,
    channel stride (W + 5)(H + 2)) inside a parent whose other elements are NaN, then -0.0 / 1e30: the same bits as
    contiguous inputs, and the parents unchanged.  NaN survives a multiplication by a zero mask and a use as zero
    padding; the second gap poison catches a read whose NaN would be discarded by a comparison."""
    plan = row.build(spec)
    rc, P, ws = _run(eng, row, spec, plan)
    _ok(eng, rc, P, ws, "contiguous")
    base = _outputs(plan, P)
    del P, ws
    for layout in bb.LAYOUTS:
        for gap in (0, 1):
            rc, P, ws = _run(eng, row, spec, plan, layout=layout, poison=1 - gap, gap=gap)
            _ok(eng, rc, P, ws, layout)
            assert bool(torch.isnan(P.inputs[0].view(torch.float32, (P.inputs[0].nbytes // 4,))).any()) == \
                (gap == 0 and layout in ("slice", "padded"))
            _assert_same_bits(base, _outputs(plan, P), f"inputs as {layout} views, gap poison {gap}")
            del P, ws


# -------------------------------------------------------------------- 6: ragged neighbours
@pytest.mark.parametrize("row,spec", RAGGED, ids=RAGGED_IDS)
def test_ragged_images_back_to_back(eng, row, spec):
    """Every per-image buffer of a ragged call in its own arena, then all images of each family back to back in one
    arena with no gap (an overrun of image i lands in image i + 1): the same bits, every guard and input intact."""
    plan = row.build(spec)
    rc, P, ws = _run(eng, row, spec, plan, offset=512)
    _ok(eng, rc, P, ws, "separate")
    base = _outputs(plan, P)
    del P, ws
    rc, P, ws = _run(eng, row, spec, plan, offset=256, poison=1, ws_fill=1, packed=True)
    _ok(eng, rc, P, ws, "packed")
    assert any(len([b for b in plan.bufs if b.group == g]) > 1 for g in {b.group for b in plan.bufs if b.group})
    _assert_same_bits(base, _outputs(plan, P), "back-to-back images")


# -------------------------------------------------------------------- 7: one byte short
@pytest.mark.parametrize("row,spec", WS_CASES, ids=WS_IDS)
def test_one_byte_short_workspace_is_refused_untouched(eng, row, spec):
    """need - 1 bytes: WN_E_WORKSPACE before any launch; outputs and workspace untouched; the message says the
    workspace is too small (with both byte counts where it gives numbers)."""
    if spec.get("shape") == bb.BIG:
        pytest.skip("the refusal is checked at the small shapes")
    plan = row.build(spec)
    need = bb.workspace_bytes(eng.lib, row, spec)
    P = bb.place(plan.bufs, 256, 1)
    for a in P.arenas:
        a.snapshot()
    ws = bb.Arena("workspace", need - 1, 768, seed=78).poison("u8", 1)
    ws.snapshot()
    before = eng.launch_count
    torch.cuda.synchronize()
    rc = plan.issue(P, ws.ptr, need - 1, bb._stream(), eng)
    msg = _error(eng)
    assert rc == bb.WN_E_WORKSPACE, f"code {rc}: {msg}"
    assert eng.launch_count == before
    bb.check(P.arenas + [ws])
    assert "too small" in msg, msg
    nums = re.search(r"(\d+) < (\d+)", msg)
    if nums:
        assert (int(nums.group(1)), int(nums.group(2))) == (need - 1, need), msg


PAIR_CASES = [(r, s) for r, s in WS_CASES if len(r.calls) == 2]


@pytest.mark.parametrize("row,spec", PAIR_CASES, ids=[f"{r.name}-{bb.spec_id(s)}" for r, s in PAIR_CASES])
def test_backward_of_a_pair_refuses_one_byte_short_untouched(eng, row, spec):
    """The forward of a pair with its full workspace, then the backward told the workspace is need - 1 bytes:
    WN_E_WORKSPACE before any launch, and the gradients and the forward's workspace untouched."""
    plan = row.build(spec)
    need = bb.workspace_bytes(eng.lib, row, spec)
    P = bb.place(plan.bufs, 512, 0)
    ws = bb.Arena("workspace", need, 256, seed=79).poison("u8", 0)
    rc = plan.issue(P, ws.ptr, need, bb._stream(), eng, stage="forward")
    assert rc == 0, _error(eng)
    torch.cuda.synchronize()
    for a in P.arenas + [ws]:
        a.snapshot()
    before = eng.launch_count
    rc = plan.issue(P, ws.ptr, need - 1, bb._stream(), eng, stage="backward")
    msg = _error(eng)
    assert rc == bb.WN_E_WORKSPACE, f"code {rc}: {msg}"
    assert eng.launch_count == before
    bb.check(P.arenas + [ws])
    assert "too small" in msg, msg
    nums = re.search(r"(\d+) < (\d+)", msg)
    if nums:
        assert (int(nums.group(1)), int(nums.group(2))) == (need - 1, need), msg


@pytest.mark.parametrize("row,spec", [(r, s) for r in bb.ROWS for s in r.rejected],
                         ids=[f"{r.name}-{bb.spec_id(s)}" for r in bb.ROWS for s in r.rejected])
def test_rejected_modes_are_refused_untouched(eng, row, spec):
    plan = row.build(spec)
    P = bb.place(plan.bufs, 0, 0)
    for a in P.arenas:
        a.snapshot()
    ws = bb.Arena("workspace", 1 << 20, 0).poison("u8", 0)
    ws.snapshot()
    before = eng.launch_count
    rc = plan.issue(P, ws.ptr, 1 << 20, bb._stream(), eng)
    assert rc == bb.WN_E_UNSUPPORTED, f"code {rc}: {_error(eng)}"
    assert eng.launch_count == before
    bb.check(P.arenas + [ws])


# -------------------------------------------------------------------- 5: selective writes
def _full_and_subset(eng, row, full_spec, sub_spec):
    plans = [row.build(s) for s in (full_spec, sub_spec)]
    outs = []
    for k, (s, plan) in enumerate(zip((full_spec, sub_spec), plans)):
        rc, P, ws = _run(eng, row, s, plan, offset=256 * k, poison=k)
        _ok(eng, rc, P, ws, bb.spec_id(s))
        outs.append(_outputs(plan, P))
    return outs


@pytest.mark.parametrize("stack,which,gin", [("cmg", 0, (True, False, True, False)), ("cmg", 0, (False,) * 4),
                                             ("refiner", 1, (False, True)), ("refiner", 2, (True, False))])
def test_submodule_backward_writes_only_its_own_entries(eng, stack, which, gin):
    """grads entries the stack does not own, given as NaN-filled guarded arenas instead of NULL, stay untouched, and
    input gradients left NULL change nothing else: the owned entries and the requested input gradients equal those
    of the call with NULL foreign entries and every input gradient requested."""
    row = bb.ROW["confidence_maps_train" if stack == "cmg" else "refine_train"]
    spec = dict(shape=(2, 37, 53), stack=stack, which=which)
    full, sub = _full_and_subset(eng, row, spec, dict(spec, gin=gin, foreign=True))
    _assert_same_bits({k: full[k] for k in sub}, sub, "owned entries with arenas elsewhere and some input grads NULL")


@pytest.mark.parametrize("stack,which", [("cmg", 0), ("refiner", 0), ("refiner", 2)])
def test_submodule_backward_tiled_writes_only_its_own_entries(eng, stack, which):
    """The windowed sub-module backwards: foreign grads entries as guarded NaN arenas stay untouched."""
    row = bb.ROW["confidence_maps_backward_tiled" if stack == "cmg" else "refine_backward_tiled"]
    spec = dict(shape=(2, 37, 53), tile=(23, 29), mpp=bb.pass_pixels(2, 37, 53, (23, 29)), stack=stack, which=which)
    plan = row.build(spec)
    shapes = bb.param_shapes()
    foreign = [i for i in range(bb.NUM_PARAMS) if i not in bb.own_params(stack, which)]
    plan.bufs += [bb.Buf(f"grads.{i}", "f32", shapes[i], "in", torch.full(shapes[i], float("nan"))) for i in foreign]
    rc, P, ws = _run(eng, row, spec, plan, offset=512, poison=1)
    _ok(eng, rc, P, ws, "foreign arenas")
    base_plan = row.build(spec)
    rc2, P2, ws2 = _run(eng, row, spec, base_plan)
    _ok(eng, rc2, P2, ws2, "NULL")
    got = {k: v for k, v in _outputs(plan, P).items()}
    _assert_same_bits(_outputs(base_plan, P2), got, "owned entries with NULL or arenas elsewhere")


PRE_SUBSETS = [tuple(k for i, k in enumerate(bb.PRE_OUTS) if m >> i & 1) for m in range(1, 1 << len(bb.PRE_OUTS))]


_PRE_FULL = {}


@pytest.mark.parametrize("outs", PRE_SUBSETS, ids=["+".join(o) for o in PRE_SUBSETS])
def test_preprocess_output_subsets(eng, outs):
    """wn_preprocess_u8 with each of the 127 non-empty output subsets, the others NULL: the outputs given equal those
    of the call with all seven, and nothing around them moves.  24 x 8 takes the 4-pixel vector path, 25 x 9 not."""
    assert len(PRE_SUBSETS) == 127
    row = bb.ROW["preprocess_u8"]
    k = PRE_SUBSETS.index(outs)
    for shape in [(2, 25, 9), (1, 24, 8)]:
        if shape not in _PRE_FULL:
            plan = row.build(dict(shape=shape))
            rc, P, ws = _run(eng, row, dict(shape=shape), plan)
            _ok(eng, rc, P, ws, "all outputs")
            _PRE_FULL[shape] = _outputs(plan, P)
        spec = dict(shape=shape, outs=outs)
        sub_plan = row.build(spec)
        rc, P, ws = _run(eng, row, spec, sub_plan, offset=256 * (k % 4), poison=1, ws_fill=k % 2)
        _ok(eng, rc, P, ws, f"outputs {outs}")
        _assert_same_bits({o: _PRE_FULL[shape][o] for o in outs}, _outputs(sub_plan, P), f"preprocess subset {outs}")


@pytest.mark.parametrize("name,spec", [
    ("enhance_u8", dict(shape=(2, 37, 53), mode=m)) for m in bb.MODES] + [
    ("enhance_u8_tiled", dict(shape=(2, 37, 53), tile=(23, 29), mpp=bb.pass_pixels(2, 37, 53, (23, 29)), mode=m))
    for m in bb.TC_MODES] + [
    ("enhance_u8_ragged", dict(sizes=bb.RAGGED[0], tile=(37, 53), mpp=bb.ragged_pass_pixels(bb.RAGGED[0], (37, 53)),
                               mode=m)) for m in bb.TC_MODES])
def test_enhance_u8_result_does_not_depend_on_out_f32(eng, name, spec):
    """The uint8 image is the same with and without out_f32 (for a ragged call: with it NULL for some images)."""
    row = bb.ROW[name]
    if name == "enhance_u8_ragged":
        m = len(spec["sizes"])
        variants = [dict(spec, f32=[True] * m), dict(spec, f32=[False] * m), dict(spec, f32=[k % 2 == 1 for k in range(m)])]
    else:
        variants = [dict(spec, f32=True), dict(spec, f32=False)]
    res = []
    for k, s in enumerate(variants):
        plan = row.build(s)
        rc, P, ws = _run(eng, row, s, plan, offset=256 * k, poison=k % 2, ws_fill=k % 2)
        _ok(eng, rc, P, ws, bb.spec_id(s))
        res.append(_outputs(plan, P))
    for r in res[1:]:
        u8 = [k for k in r if k.startswith("out_u8")]
        _assert_same_bits({k: res[0][k] for k in u8}, {k: r[k] for k in u8}, "uint8 output")
        f32 = [k for k in r if k.startswith("out_f32")]
        _assert_same_bits({k: res[0][k] for k in f32}, {k: r[k] for k in f32}, "fp32 output")


def test_ragged_training_with_some_input_gradients_null(eng):
    row = bb.ROW["train_ragged"]
    spec = dict(sizes=bb.TRAIN_RAGGED[0])
    full, sub = _full_and_subset(eng, row, spec, dict(spec, null_gin=("gin.0.1", "gin.1.0", "gin.1.3", "gin.2.2")))
    _assert_same_bits({k: full[k] for k in sub}, sub, "requested outputs")


# -------------------------------------------------------------------- 8: the range guard's re-run
def _stress_engine():
    from test_gpu_parity import _scaled_refiner_sd
    from oracle import forward as ofw
    from waternet_b200.engine import new_engine
    e = new_engine("cuda:0")
    sd = _scaled_refiner_sd(400.0)
    params = [sd[k].float() for k, _ in ofw.state_dict_spec()]
    return e, params


def _images(sizes, seed=5):
    from oracle import forward as ofw
    return [torch.from_numpy(np.ascontiguousarray(ofw.synthetic_image(seed + i, h, w, "smooth")))
            for i, (h, w) in enumerate(sizes)]


GUARD_CASES = [("enhance_u8", dict(shape=(3, 40, 56), mode=bb.DEFAULT, f32=True)),
               ("enhance_u8_peers", dict(shape=(3, 40, 56), mode=bb.DEFAULT, f32=True, peers=2)),
               ("forward", dict(shape=(3, 40, 56), mode=bb.DEFAULT)),
               ("forward_tiled", dict(shape=(3, 40, 56), tile=(23, 29), mpp=bb.pass_pixels(3, 40, 56, (23, 29)),
                                      mode=bb.DEFAULT)),
               ("enhance_u8_tiled", dict(shape=(3, 40, 56), tile=(23, 29), mpp=bb.pass_pixels(3, 40, 56, (23, 29)),
                                         mode=bb.DEFAULT, f32=True)),
               ("enhance_u8_ragged", dict(sizes=[(40, 56), (1, 1), (37, 53)], tile=(37, 53),
                                          mpp=bb.ragged_pass_pixels([(40, 56), (37, 53)], (37, 53)), mode=bb.DEFAULT,
                                          f32=[True, False, True])),
               ("forward_ragged", dict(sizes=[(40, 56), (1, 1), (37, 53)], tile=(37, 53),
                                       mpp=bb.ragged_pass_pixels([(40, 56), (37, 53)], (37, 53)), mode=bb.DEFAULT))]


@pytest.mark.parametrize("name,spec", GUARD_CASES, ids=[n for n, _ in GUARD_CASES])
def test_range_guard_rerun_stays_inside_the_buffers(name, spec):
    """Weights whose activations leave the e4m3 range: the default mode's bf16x3 re-run writes every output a second
    time.  Every guard holds, the two poisons give the same bits, and the result is the bf16x3 call's."""
    e, params = _stress_engine()
    row = bb.ROW[name]
    plan = row.build(spec)
    if "sizes" in spec:
        imgs = _images(spec["sizes"])
    else:
        n, h, w = spec["shape"]
        imgs = _images([(h, w)] * n)
    pre = [e.preprocess(t.cuda()[None]) for t in imgs]
    for b in plan.bufs:   # smooth images (random noise does not leave the e4m3 range)
        if b.role != "in":
            continue
        key, _, idx = b.name.partition(".")
        if key == "rgb":
            b.data = torch.stack(imgs).reshape(b.shape) if not idx else imgs[int(idx)].reshape(b.shape)
        elif key in bb.IN4:
            b.data = (torch.cat([p[key] for p in pre]) if not idx else pre[int(idx)][key]).cpu().reshape(b.shape)
    outs = []
    for k in range(2):
        e.pack_weights(params)   # clears the sticky flag: each call trips the guard and re-runs itself
        rc, P, ws = _run(e, row, spec, plan, offset=256 * k + 256, poison=k, ws_fill=k)
        _ok(e, rc, P, ws, f"poison {k}")
        assert e.f8_overflowed(), "the stress weights did not trip the range guard"
        outs.append(_outputs(plan, P))
    _assert_same_bits(outs[0], outs[1], "the two poisons")
    plain = row.build(dict(spec, mode=bb.BF16X3))
    for b, c in zip(plain.bufs, plan.bufs):
        b.data = c.data
    e.pack_weights(params)
    rc, P, ws = _run(e, row, dict(spec, mode=bb.BF16X3), plain)
    _ok(e, rc, P, ws, "bf16x3")
    _assert_same_bits(outs[0], _outputs(plain, P), "the bf16x3 call")


# -------------------------------------------------------------------- 9: peer stores of any alignment
PEER_OFFSETS = (0, 1, 2, 3, 4, 12)


PEER_CASES = [((2, 33, 47), False), ((2, 33, 47), True), ((1, 37, 53), False), ((3, 37, 53), True)]


def _peer_mirrors(e, mode, shape, multi_pass, rgb=None):
    """One wn_enhance_u8_peers call with a mirror at each of PEER_OFFSETS (mod 16), each in its own guarded arena;
    multi_pass caps a pass at one image.  Checks every guard and that every mirror holds the output."""
    n, h, w = shape
    assert (n * h * w * 3) % 96 and (n * h * w * 3) % 16
    row = bb.ROW["enhance_u8_peers"]
    spec = dict(shape=shape, mode=mode, f32=False, peers=len(PEER_OFFSETS))
    plan = row.build(spec)
    if rgb is not None:
        plan.bufs[0].data = rgb
    P = bb.place([b for b in plan.bufs if not b.name.startswith("peer")], 512, 0)
    mirrors = [bb.Arena(f"peer at {o} mod 16", n * h * w * 3, o, seed=90 + o).poison("u8", k % 2)
               for k, o in enumerate(PEER_OFFSETS)]
    for k, a in enumerate(mirrors):
        P._ptr[f"peer.{k}"] = a.ptr
        assert a.ptr % 16 == PEER_OFFSETS[k]
    need = bb.workspace_bytes(e.lib, row, spec)
    ws = bb.Arena("workspace", need, 256).poison("u8", 1)
    e.set_chunk_pixels(h * w if multi_pass else 0)
    try:
        if multi_pass:   # the tensor-core forward caps whole images per pass: one image each
            assert e.chunk_images(n, h, w) == 1 < n
        rc = plan.issue(P, ws.ptr, need, bb._stream(), e)
        torch.cuda.synchronize()
    finally:
        e.set_chunk_pixels(0)
    assert rc == 0, _error(e)
    bb.check(P.arenas + mirrors + [ws])
    out = P.views["out_u8"]
    for a in mirrors:
        assert torch.equal(a.payload, out.reshape(-1)), a.name
    return out


@pytest.mark.parametrize("mode", bb.MODES)
@pytest.mark.parametrize("shape,multi_pass", PEER_CASES)
def test_peer_mirrors_at_any_alignment(eng, mode, shape, multi_pass):
    """wn_enhance_u8_peers with six same-GPU destinations at 0, 1, 2, 3, 4 and 12 (mod 16), each in its own guarded
    arena (n*H*W*3 is a multiple of neither 96 nor 16), in one pass and in one pass per image (the fp32 mode does
    not split its batch into passes): every mirror holds the output, and nothing around it moved."""
    if multi_pass and mode == bb.FP32:
        pytest.skip("the fp32 mode runs a batch in one pass")
    _peer_mirrors(eng, mode, shape, multi_pass)


@pytest.mark.parametrize("shape,multi_pass", [c for c in PEER_CASES if c[0][0] > 1])
def test_peer_mirrors_follow_the_range_guard_rerun(shape, multi_pass):
    """The same mirrors when the default mode's range guard trips: the bf16x3 re-run and its copy kernel store the
    output a second time, to every misaligned mirror, and stay inside each."""
    e, params = _stress_engine()
    e.pack_weights(params)
    n, h, w = shape
    rgb = torch.stack(_images([(h, w)] * n))
    out = _peer_mirrors(e, bb.DEFAULT, shape, multi_pass, rgb)
    assert e.f8_overflowed(), "the stress weights did not trip the range guard"
    e.pack_weights(params)
    want = e.enhance(rgb.cuda(), mode=bb.BF16X3)
    assert torch.equal(out, want)
