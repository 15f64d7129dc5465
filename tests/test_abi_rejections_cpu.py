"""Without a GPU: every argument check of the C ABI returns what tests/golden/abi_rejections.json records.

The cases come from _lib._SIGNATURES and the parameter names of include/waternet_b200.h, so a new entry point is
covered without a hand-written list.  From one base call per entry point (fake device addresses, real host arrays,
small valid ints), each case changes one thing: a pointer becomes NULL, a device pointer inside a host array becomes
NULL, an int becomes 0, -1 or one past a limit the header states.  A host array is changed at its first and last
entry and at the boundaries of the sub-modules' parameter gradients; a ragged table at its last image.  Each call runs
with a NULL handle and with a stand-in handle: a zero-filled host buffer, i.e. a handle whose weights were never
packed.  Recorded per case: a workspace function's return value; a call's return code, with wn_last_error() when the
code is a validation code.  The table stores, per entry point and handle, the number of cases and the most common
record, then every case whose record differs from it.

Checks that run after "wn_pack_weights has not been called" are not reached with the stand-in.  Calls that pass every
check reach the CUDA runtime; on a machine without a device they return WN_E_CUDA.  With a device they would launch
kernels on fake addresses, so the stand-in half runs only where no device is visible.

Record the table from a library: ``WATERNET_B200_LIB=<lib> python tests/test_abi_rejections_cpu.py --record <json>``.
"""
import collections
import ctypes
import json
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from waternet_b200 import _lib  # noqa: E402

GOLDEN_PATH = os.path.join(ROOT, "tests", "golden", "abi_rejections.json")

# handle lifecycle, peer memory, raw stream operations and the host table builder take no checked arguments of a call
EXCLUDED = {"wn_create", "wn_destroy", "wn_memcpy_async", "wn_stream_write_value32", "wn_stream_wait_value32",
            "wn_build_tables_host", "wn_abi_version", "wn_last_error"}
VALUE_CALLS = {"wn_launch_count", "wn_forward_chunk_images", "wn_f8_overflowed"}  # return a value, not a code
VALIDATION_CODES = (-1, -3, -4, -5)  # WN_E_INVALID, WN_E_STATE, WN_E_WORKSPACE, WN_E_UNSUPPORTED

FAKE = 0x10000  # a non-null device address; no case that passes every check runs where a device is visible
CAP = 65536     # host arrays hold this many entries, so a call with n one past its limit never reads past them
N = 2           # images of the base call
BIG = 0x7fffffff // 3 // 16 + 1  # with the other side 16: H x W one past 0x7fffffff / 3
SIZE_MAX = (1 << 64) - 1

# base value and mutations of each int parameter, by name
INTS = {
    "n": (N, (0, -1, 65536)),
    **{k: (16, (0, -1, BIG)) for k in ("h", "w", "height", "width", "dst_h", "dst_w")},
    "tile_h": (8, (0, -1)), "tile_w": (8, (0, -1)),
    "max_pass_pixels": (0, (-1, (8 << 20) + 1)),  # one past the training and VGG caps
    "mode": (-1, (0, 7)),
    "which": (0, (-1, 3)),
    "stack": (0, (-1, 2)),
    "layer": (0, (-1, 11)),
    "buffer": (14, (0, -1, 25)),
    "n_peers": (1, (0, -1, 16)),
    "swap_rb": (0, (-1,)),
    "on": (1, (0, -1)),
    "max_pixels": (0, (-1,)),
    "workspace_bytes": (1 << 40, (0, SIZE_MAX)), "ws_bytes": (1 << 40, (0, SIZE_MAX)),
}
# device-pointer arrays on the host: the entries whose NULL a case tries
PTR_ARRAYS = {"params": (0, _lib.NUM_PARAMS - 1), "grads": (0, 15, 16, 21, 22, 27, 28, 33), "input_grads": (0, 3),
              "input_grads_host": (0, 4 * N - 1), "grad_out_host": (0, N - 1), "src_dev": (0, N - 1), "peer_out": (0,)}
SIZE_ARRAYS = ("heights_host", "widths_host", "src_h", "src_w")


def _param_names():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "waternet_b200.h")).read(), flags=re.S)
    names = {}
    for fn, params in re.findall(r"\b(wn_\w+)\s*\(([^)]*)\)\s*;", text):
        names[fn] = [] if params.strip() == "void" else \
            [re.search(r"(\w+)\s*(\[[^\]]*\]\s*)*$", p.strip()).group(1) for p in params.split(",")]
    return names


class _Args:
    """The base arguments of one entry point, in host buffers that outlive the call, and one mutation of them."""

    def __init__(self, fn, names, argtypes):
        self.fn, self.names, self.types = fn, names, argtypes
        self.vals = [self.base(i) for i in range(len(names))]

    def base(self, i):
        name, t = self.names[i], self.types[i]
        if t is ctypes.c_void_p:
            return None if name == "stream" else FAKE
        if t is ctypes.POINTER(ctypes.c_int64):
            arr = (ctypes.c_int64 * 16)(*[3 * 16 * 16, 16 * 16, 16, 1] * 4)
        elif t is ctypes.POINTER(ctypes.c_void_p):
            arr = (ctypes.c_void_p * CAP)(*[FAKE] * CAP)
        elif t is ctypes.POINTER(ctypes.c_int):
            arr = (ctypes.c_int * CAP)(*[16] * CAP) if name in SIZE_ARRAYS else (ctypes.c_int * 64)()
        elif t is ctypes.POINTER(ctypes.c_float):
            arr = (ctypes.c_float * 64)()
        elif t in (ctypes.POINTER(_lib.RaggedImage), ctypes.POINTER(_lib.RaggedTensors)):
            arr = _images(t._type_)
        else:
            return INTS[name][0]
        return arr

    def cases(self):
        """(description, index, value or None, element mutation or None) of every case."""
        yield "base", None, None, None
        for i, (name, t) in enumerate(zip(self.names, self.types)):
            if name == "stream":
                continue
            if t in (ctypes.c_int, ctypes.c_longlong, ctypes.c_size_t):
                for v in INTS[name][1]:
                    yield f"{name}={v}", i, v, None
                continue
            yield f"{name}=NULL", i, "null", None
            if t is ctypes.POINTER(ctypes.c_void_p):
                entries = (0, _lib.VGG_NUM_PARAMS - 1) if self.fn == "wn_vgg_pack_weights" else PTR_ARRAYS[name]
                for k in entries:
                    yield f"{name}[{k}]=NULL", i, None, (k, None, None)
            elif name in SIZE_ARRAYS:
                for v in (0, -1, BIG):
                    yield f"{name}[{N - 1}]={v}", i, None, (N - 1, None, v)
            elif t in (ctypes.POINTER(_lib.RaggedImage), ctypes.POINTER(_lib.RaggedTensors)):
                for field, ftype in t._type_._fields_:
                    if ftype is ctypes.c_void_p:
                        yield f"{name}[{N - 1}].{field}=NULL", i, None, (N - 1, field, None)
                    elif ftype is ctypes.c_int:
                        for v in (0, -1, BIG):
                            yield f"{name}[{N - 1}].{field}={v}", i, None, (N - 1, field, v)


def _images(struct):
    arr = (struct * CAP)()
    for e in arr:
        for field, ftype in struct._fields_:
            if ftype is ctypes.c_void_p:
                setattr(e, field, FAKE)
        e.height, e.width = 16, 16
        if struct is _lib.RaggedTensors:
            e.in_strides[:] = [3 * 16 * 16, 16 * 16, 16, 1] * 4
    return arr


def _run(lib, fn, args, half):
    """Every case of ``fn`` with the handle of ``half`` ("none": no handle parameter) -> {case id: record}."""
    f = getattr(lib, fn)
    out = {}
    for desc, i, value, elem in args.cases():
        vals = list(args.vals)
        standin = None
        if half != "none":
            if half == "standin":  # a fresh never-packed handle per case: calls write into the handle
                standin = ctypes.create_string_buffer(64 * 1024)
                vals[0] = ctypes.addressof(standin)
            else:
                vals[0] = None
        if i is not None and i == 0 and half != "none" and value == "null":
            continue  # the handle's NULL is the "null" half
        if elem is not None:  # mutated in place and restored after the call
            k, field, v = elem
            entry = vals[i] if field is None else vals[i][k]
            key = k if field is None else field
            old = entry[key] if field is None else getattr(entry, key)
            if field is None:
                entry[key] = v
            else:
                setattr(entry, key, v)
        elif value == "null":
            vals[i] = None
        elif value is not None:
            vals[i] = value
        rc = f(*vals)
        if elem is not None:
            if field is None:
                entry[key] = old
            else:
                setattr(entry, key, old)
        if fn.endswith("_workspace_bytes") or fn in VALUE_CALLS:
            rec = [int(rc)]
        elif rc in VALIDATION_CODES:
            rec = [rc, lib.wn_last_error().decode()]
        else:
            rec = [rc]
        out[f"{fn}|{half}|{desc}"] = rec
        del standin
    return out


def _table(lib, halves):
    names = _param_names()
    res = {}
    for fn, (_, argtypes) in _lib._SIGNATURES.items():
        if fn in EXCLUDED or fn.startswith("wn_peer_"):
            continue
        assert fn in names, f"{fn} is not declared in include/waternet_b200.h"
        assert len(names[fn]) == len(argtypes), fn
        has_handle = argtypes and argtypes[0] is ctypes.c_void_p and names[fn][0] == "h"
        for half in (halves if has_handle else ("none",)):
            res.update(_run(lib, fn, _Args(fn, names[fn], argtypes), half))
    return res


@pytest.fixture(scope="module")
def lib():
    from waternet_b200 import build
    build.build()
    return _lib.load()


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN_PATH) as f:
        return json.load(f)


def _groups(table):
    """{case id: record} -> {"<fn>|<half>": {case: record}}"""
    out = {}
    for k, v in table.items():
        fn, half, case = k.split("|", 2)
        out.setdefault(f"{fn}|{half}", {})[case] = v
    return out


def _compress(table):
    """Per entry point and handle: "<fn>|<half>|*" -> {"cases": count, "else": the most common record}, then the id
    and record of every case whose record differs from it."""
    out = {}
    for g, cases in _groups(table).items():
        common = json.loads(collections.Counter(json.dumps(v) for v in cases.values()).most_common(1)[0][0])
        out[f"{g}|*"] = {"cases": len(cases), "else": common}
        out.update({f"{g}|{c}": v for c, v in cases.items() if v != common})
    return out


def _compare(got, golden, half):
    want = {g: cases for g, cases in _groups(golden).items() if g.split("|")[1] == half}
    assert want, f"the golden table has no {half} cases"
    got = _groups(got)
    assert sorted(got) == sorted(want), "the entry points differ from the golden table's"
    diff = []
    for g, cases in got.items():
        common = want[g].pop("*")
        assert len(cases) == common["cases"] and set(want[g]) <= set(cases), f"{g}: the cases differ from the table's"
        diff += [f"{g}|{c}: {v} != {want[g].get(c, common['else'])}" for c, v in cases.items()
                 if v != want[g].get(c, common["else"])]
    assert not diff, f"{len(diff)} cases differ:\n" + "\n".join(diff[:40])


def test_workspace_functions_return_what_they_returned(lib, golden):
    _compare(_table(lib, ()), golden, "none")


def test_calls_with_a_null_handle_reject_as_before(lib, golden):
    _compare({k: v for k, v in _table(lib, ("null",)).items() if "|none|" not in k}, golden, "null")


@pytest.mark.skipif(torch.cuda.is_available(), reason="a call that passed its checks would launch on fake addresses")
def test_calls_with_an_unpacked_handle_reject_as_before(lib, golden):
    _compare({k: v for k, v in _table(lib, ("standin",)).items() if "|none|" not in k}, golden, "standin")


if __name__ == "__main__":
    if len(sys.argv) != 3 or sys.argv[1] != "--record":
        sys.exit("usage: WATERNET_B200_LIB=<lib> python tests/test_abi_rejections_cpu.py --record <json>")
    if torch.cuda.is_available():
        sys.exit("record without a visible device: the stand-in half would launch on fake addresses")
    table = _table(_lib.load(), ("null", "standin"))
    rows = _compress(table)
    with open(sys.argv[2], "w") as f:  # one case per line
        f.write("{\n" + ",\n".join(f"{json.dumps(k)}: {json.dumps(rows[k])}" for k in sorted(rows)) + "\n}\n")
    print(f"{len(table)} cases, {len(rows)} rows -> {sys.argv[2]}")
