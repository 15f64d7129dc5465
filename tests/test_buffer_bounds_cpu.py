"""Without a GPU: the buffer-bounds table covers every entry point of the header that takes a workspace or writes
device memory, the workspace functions agree with the table, and the arena helper reports what it should."""
import os

import pytest
import torch

import buffer_bounds as bb
from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import _lib, build
    build.build()
    return _lib.load()


def _header():
    with open(os.path.join(ROOT, "include", "waternet_b200.h")) as f:
        return bb.header_functions(f.read())


def test_every_writing_entry_point_is_in_the_table_or_excluded():
    funcs = _header()
    assert len(funcs) > 40
    covered = {c for r in bb.ROWS for c in r.calls}
    writers = {name for name, params in funcs.items() if bb.writes_device_memory(params)}
    missing = sorted(writers - covered - set(bb.EXCLUDED))
    assert not missing, f"entry points without a buffer-bounds row or a named exclusion: {missing}"
    assert covered <= set(funcs), f"rows name undeclared functions: {sorted(covered - set(funcs))}"
    # the exclusions name real writers, and no row is also excluded
    assert set(bb.EXCLUDED) <= writers and not set(bb.EXCLUDED) & covered
    for r in bb.ROWS:
        if r.ws:
            assert r.ws in funcs and "workspace_bytes" in r.ws


def test_writer_detection():
    assert bb.writes_device_memory(["wn_handle* h", "const float* x", "void* workspace", "size_t workspace_bytes"])
    assert bb.writes_device_memory(["wn_handle* h", "const float* x", "float* out"])
    assert bb.writes_device_memory(["wn_handle* h", "float* const* grads"])
    assert bb.writes_device_memory(["wn_handle* h", "uint8_t* const* peer_out"])
    assert not bb.writes_device_memory(["wn_handle* h", "const float* const* params", "void* stream"])
    assert not bb.writes_device_memory(["const wn_handle* h", "int n"])


def test_rows_list_their_buffers():
    for r in bb.ROWS:
        assert r.specs, r.name
        for spec in r.specs[:2]:
            plan = r.build(spec)
            names = {b.name for b in plan.bufs}
            assert len(names) == len(plan.bufs), f"{r.name}: duplicate buffer names"
            for b in plan.bufs:
                if b.role == "in":
                    assert b.data is not None and tuple(b.data.shape) == b.shape, (r.name, b.name)
                    assert b.name.split(".")[0] in r.inputs + r.optional, (r.name, b.name)
                else:
                    assert b.name.split(".")[0] in r.outputs + r.optional, (r.name, b.name)


@pytest.mark.parametrize("row", [r for r in bb.ROWS if r.ws], ids=lambda r: r.name)
def test_workspace_functions_agree_with_the_table(lib, row):
    for spec in row.specs:
        assert bb.workspace_bytes(lib, row, spec) > 0, f"{row.name} {bb.spec_id(spec)}"
    for spec in row.rejected:
        assert bb.workspace_bytes(lib, row, spec) == 0, f"{row.name} rejects {bb.spec_id(spec)}"


def test_tiled_specs_run_many_passes_with_a_partial_last_one():
    from waternet_b200.engine import tile_geometry
    for (n, h, w), tile in bb.TILES:
        g = tile_geometry(h, w, *tile)
        windows = n * g["ny"] * g["nx"]
        per = bb.pass_pixels(n, h, w, tile) // (g["win_h"] * g["win_w"])
        assert per == 3
        if windows > 3:
            assert windows % per or (n, h, w) == (300, 5, 7), ((n, h, w), tile, windows)


# ---------------------------------------------------------------------------------------------- the arena helper
@pytest.mark.parametrize("offset", bb.START_OFFSETS + (1, 13))
def test_arena_places_the_payload_at_the_offset(offset):
    a = bb.Arena("buf", 1000, offset, seed=3, device="cpu")
    assert a.ptr % 1024 == offset
    assert a.start >= bb.GUARD and a.raw.numel() - a.end >= bb.GUARD
    assert a.end - a.start == 1000
    a.poison("u8", 1)
    assert bool((a.payload == 0xFF).all())
    assert a.damage() == []


def test_arena_reports_guard_damage_with_offsets():
    a = bb.Arena("ws", 1000, 256, seed=5, device="cpu")
    a.poison("u8", 0)
    a.payload.fill_(7)                       # writes inside the payload are not damage
    assert a.damage() == []
    a.raw[a.end + 3] ^= 0xFF                  # bytes 3 and 9 after the payload's end
    a.raw[a.end + 9] ^= 0x01
    a.raw[a.start - 2] ^= 0x10                # two bytes before its start
    lines = a.damage()
    assert len(lines) == 2
    assert "front guard" in lines[0] and "offsets -2..-2" in lines[0] and "1 bytes" in lines[0]
    assert "back guard" in lines[1] and "offsets 3..9" in lines[1] and "2 bytes" in lines[1]
    with pytest.raises(AssertionError, match="ws: 2 bytes of the back guard"):
        bb.check([a])


def test_arena_snapshot_reports_payload_writes():
    a = bb.Arena("x", 64, 512, device="cpu")
    a.payload.copy_(torch.arange(64, dtype=torch.uint8))
    a.snapshot()
    a.payload[10] = 0
    a.payload[40] = 0
    (line,) = a.damage()
    assert "payload" in line and "offsets 10..40" in line


def test_poisons_differ_in_every_fp32_element():
    a = bb.Arena("out", 4 * 10, 0, device="cpu")
    a.poison("f32", 0)
    first = a.payload.clone()
    assert bool(torch.isnan(a.view(torch.float32, (10,))).all())
    a.poison("f32", 1)
    f = a.view(torch.float32, (10,))
    assert f[0].item() == 0.0 and str(f[0].item()) == "-0.0" and f[1].item() == torch.tensor(1e30).item()
    assert bool((first.view(torch.int32) != a.payload.view(torch.int32)).all())


@pytest.mark.parametrize("layout", ("contiguous",) + bb.LAYOUTS)
def test_strided_views_hold_the_values_and_poison_the_gaps(layout):
    for gap in (0, 1):
        _check_view(layout, gap)


def _check_view(layout, gap):
    """Input gaps hold poison ``gap`` (0: NaN), the outputs the other one."""
    data = torch.rand(2, 3, 5, 7)
    bufs = [bb.Buf("x", "f32", (2, 3, 5, 7), "in", data, nchw=True), bb.Buf("out", "f32", (2, 3, 5, 7), "out")]
    P = bb.place(bufs, offset=256, poison=1 - gap, layout=layout, device="cpu", gap=gap)
    v = P.views["x"]
    assert torch.equal(v, data)
    a = P.arenas[0]
    assert P.inputs == [a]
    assert bool(torch.isnan(P.views["out"]).all()) == (gap == 1)
    used = torch.zeros(a.nbytes // 4, dtype=torch.bool)
    base = (v.data_ptr() - a.ptr) // 4
    idx = torch.as_strided(torch.arange(a.nbytes // 4), v.shape, v.stride(), base)
    used[idx.flatten()] = True
    gaps = a.view(torch.float32, (a.nbytes // 4,))[~used]
    if gap == 0:
        assert bool(torch.isnan(gaps).all())
    else:
        assert all(g in (-0.0, torch.tensor(1e30).item()) for g in gaps.tolist())
    assert (layout in ("contiguous", "channels_last")) == (gaps.numel() == 0)
    if layout == "padded":
        assert v.stride() == (3 * 12 * 7, 12 * 7, 12, 1)
    assert a.damage() == []
    v[0, 0, 0, 0] = 0.5                     # a write into an input shows as payload damage
    assert any("payload" in line for line in a.damage())


def test_packed_groups_sit_back_to_back():
    bufs = [bb.Buf(f"rgb.{i}", "u8", (h, w, 3), "in", torch.full((h, w, 3), i, dtype=torch.uint8), group="rgb")
            for i, (h, w) in enumerate([(1, 1), (3, 5), (2, 2)])]
    P = bb.place(bufs, offset=768, packed=True, device="cpu")
    assert len(P.arenas) == 1 and P.arenas[0].nbytes == 3 + 45 + 12
    assert P.ptr("rgb.1") == P.ptr("rgb.0") + 3 and P.ptr("rgb.2") == P.ptr("rgb.1") + 45
    sep = bb.place(bufs, offset=768, packed=False, device="cpu")
    assert len(sep.arenas) == 3 and all(p % 1024 == 768 for p in (sep.ptr(b.name) for b in bufs))
