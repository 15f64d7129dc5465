"""Where wn_ssim_grad writes and what it reads, on the GPU, with the guarded arenas of tests/buffer_bounds.py.

The checks tests/test_metrics_native_bounds_gpu.py runs on wn_quality, for the entry point of
include/waternet_b200_ssim.h: every image's out, ref and grad and the stats buffer in guarded arenas, the workspace
exactly wn_ssim_grad_workspace_bytes; run at the four start offsets with both poisons of outputs and workspace, the
stats and gradients are the same bits, every guard and input is intact, every grad element is written, and they
equal Engine.ssim_grad on plain tensors; the images of each family back to back give the same bits; a workspace one
byte short is refused before any launch with everything untouched.
"""
import pytest
import torch

import buffer_bounds as bb

pytestmark = pytest.mark.gpu

SPECS = [dict(sizes=[(6, 6), (11, 11), (12, 13)], groups=(0, 0, 1), scales=(-0.5, -0.5, -1.0)),
         dict(sizes=[(37, 53), (6, 9), (25, 17), (64, 97)], groups=(2, 0, 2, 1), scales=(0.25, 1.0, 0.25, -2.0)),
         dict(sizes=[(130, 70)], groups=(0,), scales=(-1.0,)),
         dict(sizes=[bb.BIG[1:]], groups=(0,), scales=(-1.0,))]
IDS = [bb.spec_id(dict(sizes=s["sizes"], groups=s["groups"])) for s in SPECS]


def _plan(spec):
    from waternet_b200 import _lib as L
    sizes, groups, scales = spec["sizes"], spec["groups"], spec["scales"]
    n = len(sizes)
    bufs = [bb._f32_in(f"{k}.{i}", (3, h, w), 30 + 2 * i + j, nchw=False, group=k)
            for j, k in enumerate(("out", "ref")) for i, (h, w) in enumerate(sizes)]
    bufs += [bb._out(f"grad.{i}", "f32", (3, h, w), group="grad") for i, (h, w) in enumerate(sizes)]
    bufs.append(bb._out("stats", "u8", (n * L.QUALITY_STATS * 8,)))

    def issue(P, ws, nb, eng):
        table = (L.SSIMGradImage * n)()
        for d, (h, w), g, sc, i in zip(table, sizes, groups, scales, range(n)):
            d.out, d.ref, d.grad = P.ptr(f"out.{i}"), P.ptr(f"ref.{i}"), P.ptr(f"grad.{i}")
            d.height, d.width, d.group, d.scale = h, w, g, sc
        with torch.cuda.device(eng.device):
            return eng.lib.wn_ssim_grad(eng.handle, table, n, P.ptr("stats"), ws, nb, bb._stream())
    return bufs, issue


def _need(eng, spec):
    return eng.ssim_grad_workspace_bytes(spec["sizes"])


@pytest.fixture(scope="module")
def eng():
    from waternet_b200.engine import new_engine
    return new_engine("cuda:0")


def _run(eng, spec, offset=0, poison=0, ws_fill=0, packed=False):
    bufs, issue = _plan(spec)
    P = bb.place(bufs, offset, poison, packed=packed)
    nb = _need(eng, spec)
    ws = bb.Arena("workspace", nb, offset, seed=79).poison("u8", ws_fill)
    torch.cuda.synchronize()
    rc = issue(P, ws.ptr, nb, eng)
    torch.cuda.synchronize()
    assert rc == 0, eng.lib.wn_last_error().decode()
    bb.check(P.arenas + [ws])
    n = len(spec["sizes"])
    return [P.views["stats"].clone()] + [P.views[f"grad.{i}"].clone() for i in range(n)], bufs


def _same(a, b):
    return all(torch.equal(x.view(torch.uint8) if x.dtype != torch.uint8 else x,
                           y.view(torch.uint8) if y.dtype != torch.uint8 else y) for x, y in zip(a, b))


@pytest.mark.parametrize("spec", SPECS, ids=IDS)
def test_exact_workspace_full_writes_and_no_uninitialised_reads(eng, spec):
    results = [_run(eng, spec, off, poison=k % 2, ws_fill=(k ^ (k >> 1)) & 1)[0]
               for k, off in enumerate(bb.START_OFFSETS)]
    for k in range(1, 4):
        assert _same(results[0], results[k]), f"offset {bb.START_OFFSETS[k]} against offset 0"
    bufs, _ = _plan(spec)
    T = {b.name: b.data.cuda() for b in bufs if b.role == "in"}
    n = len(spec["sizes"])
    stats, grads = eng.ssim_grad([T[f"out.{i}"] for i in range(n)], [T[f"ref.{i}"] for i in range(n)],
                                 spec["groups"], spec["scales"])
    assert torch.equal(results[0][0], stats.reshape(-1).view(torch.uint8))
    for i in range(n):
        assert torch.equal(results[0][1 + i].reshape(-1).view(torch.uint8), grads[i].reshape(-1).view(torch.uint8))
    eng.release_workspaces()


@pytest.mark.parametrize("spec", [s for s in SPECS if len(s["sizes"]) > 1],
                         ids=[i for s, i in zip(SPECS, IDS) if len(s["sizes"]) > 1])
def test_images_back_to_back(eng, spec):
    base, _ = _run(eng, spec, offset=512)
    packed, _ = _run(eng, spec, offset=256, poison=1, ws_fill=1, packed=True)
    assert _same(base, packed)


@pytest.mark.parametrize("spec", SPECS[:3], ids=IDS[:3])
def test_one_byte_short_workspace_is_refused_untouched(eng, spec):
    bufs, issue = _plan(spec)
    need = _need(eng, spec)
    P = bb.place(bufs, 256, 1)
    for a in P.arenas:
        a.snapshot()
    ws = bb.Arena("workspace", need - 1, 768, seed=80).poison("u8", 1)
    ws.snapshot()
    before = eng.launch_count
    torch.cuda.synchronize()
    rc = issue(P, ws.ptr, need - 1, eng)
    msg = eng.lib.wn_last_error().decode()
    assert rc == bb.WN_E_WORKSPACE, f"code {rc}: {msg}"
    assert eng.launch_count == before
    bb.check(P.arenas + [ws])
    assert "too small" in msg, msg
