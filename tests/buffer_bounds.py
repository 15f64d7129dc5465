"""Where the C-ABI calls write and what they read: guarded arenas and the table of entry points they check.

Every buffer a call receives is placed in a fresh uint8 allocation of its own, ``[front guard | payload | back
guard]``, with 1 MiB guards of a seeded pseudo-random byte pattern and a payload of exactly the requested length at a
chosen start offset (mod 1024).  A store past a buffer lands in its guard, and ``Arena.damage`` reports it with its
offsets instead of corrupting someone else's tensor.  Payloads are poisoned (NaN / -0.0 and 1e30 for fp32, 0x00 / 0xFF
for bytes), so a call run twice with the two poisons gives different bits wherever it leaves an output element
unwritten or reads one it did not write.

``ROWS`` names every entry point that takes a workspace or writes device memory, with its workspace function, its
inputs (unchanged by the call), its outputs (written in full), its optional outputs and a builder that issues the raw
call through ctypes.  tests/test_buffer_bounds_gpu.py runs the rows on the GPU; tests/test_buffer_bounds_cpu.py checks,
without one, that the table covers the header and that the workspace functions agree with it.  This module imports
without a GPU.
"""
from __future__ import annotations

import ctypes
import re
from ctypes import c_int, c_int64, c_void_p
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import torch

GUARD = 1 << 20                      # bytes of guard on each side of a payload
START_OFFSETS = (0, 256, 512, 768)   # payload starts (mod 1024): torch gives 512 B alignment, the calls realign
LAYOUTS = ("slice", "channels_last", "padded")  # strided views of fp32 (N,3,H,W) inputs inside a poisoned parent

FP32, BF16X3, DEFAULT = 0, 1, -1     # WN_MODE_*
WN_E_WORKSPACE, WN_E_UNSUPPORTED = -4, -5
NUM_PARAMS, VGG_NUM_PARAMS = 34, 32

# element strides of the padded-row layout: row stride W + 5, channel stride (W + 5) * (H + 2)
PAD_W, PAD_H = 5, 2


def _pattern(n: int, seed: int, device) -> torch.Tensor:
    g = torch.Generator(device=device).manual_seed(seed)
    return torch.randint(0, 256, (n,), dtype=torch.uint8, device=device, generator=g)


def poison_(t: torch.Tensor, kind: str, which: int) -> None:
    """Fill the uint8 tensor ``t`` with poison ``which`` (0 or 1) of ``kind``: fp32 NaN, then -0.0 / 1e30
    alternating; bytes 0x00, then 0xFF.  An fp32 poison over a length that is not a multiple of 4 leaves the tail
    bytes 0xFF (a NaN pattern)."""
    if kind == "f32":
        t.fill_(0xFF)
        f = t[:t.numel() // 4 * 4].view(torch.float32)
        if which == 0:
            f.fill_(float("nan"))
        else:
            f[0::2] = -0.0
            f[1::2] = 1e30
    else:
        t.fill_(0x00 if which == 0 else 0xFF)


class Arena:
    """One fresh uint8 allocation laid out as [front guard | payload | back guard].

    ``nbytes``: the payload length, exactly (the back guard starts at payload byte ``nbytes``).  ``offset``: the
    payload's start address mod 1024.  The guards hold a pseudo-random pattern of ``seed``; the payload is left
    uninitialised until ``poison`` or a write into ``view``."""

    def __init__(self, name: str, nbytes: int, offset: int = 0, seed: int = 0, device="cuda"):
        self.name, self.nbytes, self.offset = name, int(nbytes), int(offset)
        self.raw = torch.empty(2 * GUARD + 1024 + self.nbytes, dtype=torch.uint8, device=device)
        self.start = GUARD + (self.offset - (self.raw.data_ptr() + GUARD)) % 1024
        self.end = self.start + self.nbytes
        self.raw[:self.start] = _pattern(self.start, seed, device)
        self.raw[self.end:] = _pattern(self.raw.numel() - self.end, seed + 1, device)
        self._front = self.raw[:self.start].clone()
        self._back = self.raw[self.end:].clone()
        self._snapshot = None

    @property
    def ptr(self) -> int:
        return self.raw.data_ptr() + self.start

    @property
    def payload(self) -> torch.Tensor:
        return self.raw[self.start:self.end]

    def view(self, dtype, shape, strides=None, byte_offset: int = 0) -> torch.Tensor:
        """A typed view of the payload from ``byte_offset`` (a multiple of the element size), contiguous or with
        element ``strides``."""
        size = torch.empty((), dtype=dtype).element_size()
        assert byte_offset % size == 0 and (self.ptr + byte_offset) % size == 0
        span = (self.nbytes - byte_offset) // size * size
        flat = self.raw[self.start + byte_offset:self.start + byte_offset + span].view(dtype)
        if strides is None:
            strides = torch.empty(shape, device="meta").stride()
        return flat.as_strided(tuple(shape), tuple(strides))

    def poison(self, kind: str, which: int) -> "Arena":
        poison_(self.payload, kind, which)
        return self

    def snapshot(self) -> None:
        """Remember the payload: ``damage`` then also reports every payload byte that changed."""
        self._snapshot = self.payload.clone()

    def damage(self) -> List[str]:
        """What changed outside the payload (and inside it, after ``snapshot``): one line per region with the
        first and last changed offset and the byte count.  Offsets before the payload are negative and relative to
        its start; offsets after it count from its end."""
        if self.raw.is_cuda:
            torch.cuda.synchronize(self.raw.device)
        out = []
        regions = [("front guard", self._front, 0, self.start), ("back guard", self._back, self.end, self.end)]
        if self._snapshot is not None:
            regions.append(("payload", self._snapshot, self.start, self.start))
        for what, ref, lo, origin in regions:
            diff = torch.nonzero(self.raw[lo:lo + ref.numel()] != ref).flatten()
            if diff.numel():
                first, last = int(diff[0]) + lo - origin, int(diff[-1]) + lo - origin
                rel = "payload end" if what == "back guard" else "payload start"
                out.append(f"{self.name}: {diff.numel()} bytes of the {what} changed, offsets {first}..{last} "
                           f"from the {rel} (payload {self.nbytes} bytes at {self.offset} mod 1024)")
        return out


def check(arenas) -> None:
    """Assert that no guard (and no snapshotted payload) of ``arenas`` changed."""
    bad = [line for a in arenas for line in a.damage()]
    assert not bad, "\n".join(bad)


# ---------------------------------------------------------------------------------------------- buffers of a call
@dataclass
class Buf:
    """One buffer of a call.  ``role``: "in" (must stay unchanged), "out" (written in full).  ``data``: an input's
    values (CPU).  ``group``: the per-image family of a ragged call ("rgb" for rgb.0, rgb.1, ...), laid out back to
    back in one arena in the packed layout.  ``nchw``: an fp32 (N,3,H,W) input read through element strides."""
    name: str
    kind: str
    shape: Tuple[int, ...]
    role: str
    data: Optional[torch.Tensor] = None
    group: Optional[str] = None
    nchw: bool = False

    @property
    def dtype(self):
        return torch.float32 if self.kind == "f32" else torch.uint8

    @property
    def numel(self) -> int:
        n = 1
        for s in self.shape:
            n *= s
        return n

    @property
    def nbytes(self) -> int:
        return self.numel * (4 if self.kind == "f32" else 1)


def _layout(shape, layout):
    """(parent elements, element strides, element offset) of an (N,3,H,W) view in ``layout``."""
    n, c, h, w = shape
    if layout == "contiguous":
        return n * c * h * w, (c * h * w, h * w, w, 1), 0
    if layout == "slice":
        return n * c * h * w + 74, (c * h * w, h * w, w, 1), 37
    if layout == "channels_last":
        return n * c * h * w, (h * w * c, 1, w * c, c), 0
    if layout == "padded":
        rw, ch = w + PAD_W, (w + PAD_W) * (h + PAD_H)
        return n * c * ch, (c * ch, ch, rw, 1), rw + 2
    raise ValueError(layout)


class Placed:
    """The buffers of one call in their arenas: ``ptr(name)`` (None for a buffer the call does not get),
    ``strides(name)``, the typed ``views`` and every ``arenas`` entry for ``check``."""

    def __init__(self):
        self.views: Dict[str, torch.Tensor] = {}
        self._ptr: Dict[str, int] = {}
        self._strides: Dict[str, Tuple[int, ...]] = {}
        self.arenas: List[Arena] = []
        self.inputs: List[Arena] = []

    def ptr(self, name):
        return self._ptr.get(name)

    def strides(self, name):
        return self._strides[name]


def place(bufs, offset=0, poison=0, layout="contiguous", packed=False, seed=0, device="cuda", gap=None) -> Placed:
    """Put ``bufs`` into fresh guarded arenas with payloads at ``offset`` (mod 1024).  Output payloads hold poison
    ``poison``, the unused parts of input parents poison ``gap`` (default: ``poison``; 0 is NaN for fp32); inputs get
    their values and are snapshotted, so that ``check`` also catches a write into an input.  ``layout``: the view
    of the fp32 (N,3,H,W) inputs.  ``packed``:
    the buffers of each ragged group back to back, with no gap, in one arena."""
    pl = Placed()
    groups: Dict[str, List[Buf]] = {}
    for b in bufs:
        if packed and b.group:
            groups.setdefault(b.group, []).append(b)
        else:
            groups[b.name] = [b]
    for k, (gname, members) in enumerate(groups.items()):
        spans = []
        total = 0
        for b in members:
            lay = layout if b.nchw else "contiguous"
            elems, strides, eoff = _layout(b.shape, lay) if len(b.shape) == 4 else (b.numel, None, 0)
            size = 4 if b.kind == "f32" else 1
            spans.append((b, total, strides, eoff))
            total += elems * size
        a = Arena(gname, total, offset, seed=seed + 2 * k, device=device)
        is_input = any(b.role == "in" for b in members)
        a.poison(members[0].kind, poison if gap is None or not is_input else gap)
        for b, base, strides, eoff in spans:
            size = 4 if b.kind == "f32" else 1
            v = a.view(b.dtype, b.shape, strides, base + eoff * size)
            if b.role == "in":
                v.copy_(b.data)
            pl.views[b.name] = v
            pl._ptr[b.name] = v.data_ptr()
            pl._strides[b.name] = tuple(v.stride())
        if is_input:
            a.snapshot()
            pl.inputs.append(a)
        pl.arenas.append(a)
    return pl


# ------------------------------------------------------------------------------------------------ the entry points
@dataclass
class Plan:
    """One argument set of a row: its buffers, and ``issue(P, ws_ptr, ws_bytes, stream, engine) -> rc`` on the
    engine's handle (a pair issues both calls and returns the first nonzero code; its ``stage="forward"`` or
    ``"backward"`` issues one of them)."""
    bufs: List[Buf]
    issue: Callable
    engine: Optional[Callable] = None   # (Engine, {input name: CUDA tensor}) -> {output name: tensor}


@dataclass
class Row:
    """One C-ABI entry point (or a forward / backward pair sharing a workspace).

    ``calls``: the functions the builder issues.  ``ws``: the workspace function and ``ws_args(spec)`` its
    arguments (lists become HOST int arrays).  ``inputs`` / ``outputs`` / ``optional``: buffer names or family
    prefixes ("grads", "rgb").  ``modes``: the modes the call accepts; ``rejected``: specs it refuses with
    WN_E_UNSUPPORTED (the workspace function returns 0 for them).  ``specs``: the argument sets the GPU test runs.
    ``build(spec) -> Plan``."""
    name: str
    calls: Tuple[str, ...]
    ws: Optional[str]
    ws_args: Optional[Callable]
    inputs: Tuple[str, ...]
    outputs: Tuple[str, ...]
    optional: Tuple[str, ...]
    specs: List[dict]
    build: Callable
    rejected: List[dict] = field(default_factory=list)


def workspace_bytes(lib, row: Row, spec: dict) -> int:
    args = []
    for a in row.ws_args(spec):
        args.append((c_int * max(1, len(a)))(*a) if isinstance(a, (list, tuple)) else a)
    return int(getattr(lib, row.ws)(*args))


def spec_id(spec: dict) -> str:
    parts = []
    for k, v in spec.items():
        if k == "sizes":
            v = "+".join(f"{h}x{w}" for h, w in v)
        elif isinstance(v, tuple):
            v = "x".join(map(str, v))
        parts.append(f"{k}{v}")
    return "-".join(parts)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _f32_in(name, shape, seed, nchw=True, group=None, levels=False):
    g = _gen(seed)
    data = torch.randint(0, 256, shape, generator=g).float() / 255 if levels else torch.rand(shape, generator=g)
    return Buf(name, "f32", tuple(shape), "in", data, group=group, nchw=nchw)


def _grad_in(name, shape, seed, group=None):
    return Buf(name, "f32", tuple(shape), "in", torch.randn(shape, generator=_gen(seed)) * 1e-2, group=group)


def _u8_in(name, shape, seed, group=None):
    return Buf(name, "u8", tuple(shape), "in", torch.randint(0, 256, shape, generator=_gen(seed), dtype=torch.uint8),
               group=group)


def _out(name, kind, shape, group=None):
    return Buf(name, kind, tuple(shape), "out", group=group)


def param_shapes():
    from oracle import forward as ofw
    return [s for _, s in ofw.state_dict_spec()]


def vgg_param_shapes():
    from waternet_b200.engine import VGG_CONVS
    return [s for cin, cout in VGG_CONVS for s in ((cout, cin, 3, 3), (cout,))]


def own_params(stack: str, which: int = 0) -> range:
    """Entries of ``grads`` a stack writes: all 34, the cmg's 0..15 or refiner ``which``'s 16 + 6 which .. +5."""
    return {"all": range(NUM_PARAMS), "cmg": range(16), "refiner": range(16 + 6 * which, 22 + 6 * which)}[stack]


def _grads(stack="all", which=0):
    shapes = param_shapes()
    return [_out(f"grads.{i}", "f32", shapes[i]) for i in own_params(stack, which)]


def _ptrs(P, names):
    return (c_void_p * len(names))(*[P.ptr(n) for n in names])


def _st(P, names):
    return (c_int64 * (4 * len(names)))(*[s for n in names for s in P.strides(n)])


def _stream():
    return torch.cuda.current_stream().cuda_stream


IN4 = ("x", "wb", "he", "gc")
GRADS = [f"grads.{i}" for i in range(NUM_PARAMS)]


def _lib():
    from waternet_b200 import _lib as L
    return L.load()


def _handle(eng):
    return eng.handle


# ---- shapes -------------------------------------------------------------------------------------------------------
EDGE = [(1, 1, 1), (1, 23, 7), (1, 24, 8), (1, 25, 9), (1, 23, 17), (2, 37, 53), (300, 5, 7)]
SUB_EDGE = [(1, 1, 1), (1, 24, 8), (1, 25, 17), (2, 37, 53), (300, 5, 7)]
BIG = (1, 1080, 1920)
TILES = [((2, 37, 53), (37, 53)), ((2, 37, 53), (23, 29)), ((2, 37, 53), (2, 13)), ((1, 25, 17), (23, 29)),
         ((300, 5, 7), (2, 13)), ((1, 1, 1), (2, 13))]
RAGGED = [[(1, 1), (97, 118), (23, 7), (1, 1)], [(97, 118), (1, 1), (24, 17)], [(25, 9), (1, 1)]]
RAGGED_TILES = [(37, 53), (23, 29), (23, 29)]
MODES = (FP32, BF16X3, DEFAULT)
TC_MODES = (BF16X3, DEFAULT)


def pass_pixels(n, h, w, tile, per=3):
    """A pass limit of ``per`` windows of the tiled geometry: many passes, the last one partial."""
    from waternet_b200.engine import tile_geometry
    g = tile_geometry(h, w, *tile)
    return per * g["win_h"] * g["win_w"]


def ragged_pass_pixels(sizes, tile, per=2):
    from waternet_b200.engine import tile_geometry
    big = max((tile_geometry(h, w, *tile) for h, w in sizes), key=lambda g: g["win_h"] * g["win_w"])
    return per * big["win_h"] * big["win_w"]


def _tiled_specs(modes, big=True):
    specs = [dict(shape=s, tile=t, mpp=pass_pixels(*s, t), mode=m) for m in modes for s, t in TILES]
    if big:
        specs.append(dict(shape=BIG, tile=(998, 998), mpp=0, mode=DEFAULT))
    return specs


def _ragged_specs(modes):
    return [dict(sizes=s, tile=t, mpp=ragged_pass_pixels(s, t), mode=m)
            for m in modes for s, t in zip(RAGGED, RAGGED_TILES)]


# ---- forward family ------------------------------------------------------------------------------------------------
def _ins4(shape, seed=0, levels=False):
    """x, wb, he, gc: uniform values, or 8-bit levels u / 255 (the first layer then drops its a_lo pass)."""
    return [_f32_in(k, shape, seed + i, levels=levels) for i, k in enumerate(IN4)]


def _ins_refine(shape, seed=0, levels=False):
    return [_f32_in("x", shape, seed, levels=levels), _f32_in("xbar", shape, seed + 1, levels=levels)]


def _spec_ins(spec, shape, refine=False):
    """The fp32 inputs of a spec: x, xbar of a refiner or x, wb, he, gc; 8-bit levels when spec["levels"]."""
    h, w = shape[2:]
    lv = spec.get("levels", False)
    return _ins_refine(shape, seed=h * w, levels=lv) if refine else _ins4(shape, seed=h * w, levels=lv)


def build_forward(spec, fn="wn_forward"):
    n, h, w = spec["shape"]
    shape = (n, 3, h, w)
    bufs = _spec_ins(spec, shape) + [_out("out", "f32", shape)]

    def issue(P, ws, nb, stream, eng):
        return getattr(_lib(), fn)(_handle(eng), *[P.ptr(k) for k in IN4], _st(P, IN4), P.ptr("out"), n, h, w,
                                   spec["mode"], ws, nb, stream)

    def engine(eng, T):
        f = {"wn_forward": eng.forward, "wn_confidence_maps": eng.confidence_maps}[fn]
        return {"out": f(*[T[k] for k in IN4], mode=spec["mode"])}
    return Plan(bufs, issue, engine)


def build_refine(spec):
    n, h, w = spec["shape"]
    shape, which = (n, 3, h, w), spec["which"]
    bufs = _spec_ins(spec, shape, True) + [_out("out", "f32", shape)]

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_refine(_handle(eng), which, P.ptr("x"), P.ptr("xbar"), _st(P, ("x", "xbar")), P.ptr("out"),
                                n, h, w, spec["mode"], ws, nb, stream)
    return Plan(bufs, issue, lambda eng, T: {"out": eng.refine(which, T["x"], T["xbar"], mode=spec["mode"])})


def build_forward_tiled(spec, fn="wn_forward_tiled"):
    n, h, w = spec["shape"]
    shape, (th, tw), mpp = (n, 3, h, w), spec["tile"], spec["mpp"]
    refine = fn == "wn_refine_tiled"
    names = ("x", "xbar") if refine else IN4
    bufs = _spec_ins(spec, shape, refine) + [_out("out", "f32", shape)]

    def issue(P, ws, nb, stream, eng):
        lead = (spec["which"],) if refine else ()
        return getattr(_lib(), fn)(_handle(eng), *lead, *[P.ptr(k) for k in names], _st(P, names), P.ptr("out"),
                                   n, h, w, th, tw, mpp, spec["mode"], ws, nb, stream)

    def engine(eng, T):
        kw = dict(tile=(th, tw), mode=spec["mode"], max_pass_pixels=mpp)
        if refine:
            return {"out": eng.refine_tiled(spec["which"], T["x"], T["xbar"], **kw)}
        f = eng.forward_tiled if fn == "wn_forward_tiled" else eng.confidence_maps_tiled
        return {"out": f(*[T[k] for k in IN4], **kw)}
    return Plan(bufs, issue, engine)


def _ragged_tensors(P, sizes, out=True):
    from waternet_b200 import _lib as L
    table = (L.RaggedTensors * len(sizes))()
    for i, (h, w) in enumerate(sizes):
        d = table[i]
        names = [f"{k}.{i}" for k in IN4]
        d.x, d.wb, d.he, d.gc = (P.ptr(k) for k in names)
        d.in_strides[:] = [s for k in names for s in P.strides(k)]
        d.out = P.ptr(f"out.{i}") if out else None
        d.height, d.width = h, w
    return table


def _ragged_ins(sizes, seed=0, levels=False):
    return [_f32_in(f"{k}.{i}", (1, 3, h, w), seed + 10 * i + j, group=k, levels=levels)
            for i, (h, w) in enumerate(sizes) for j, k in enumerate(IN4)]


def build_forward_ragged(spec):
    sizes, (th, tw), mpp = spec["sizes"], spec["tile"], spec["mpp"]
    bufs = _ragged_ins(sizes, levels=spec.get("levels", False))
    bufs += [_out(f"out.{i}", "f32", (1, 3, h, w), group="out") for i, (h, w) in enumerate(sizes)]

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_forward_ragged(_handle(eng), _ragged_tensors(P, sizes), len(sizes), th, tw, mpp,
                                        spec["mode"], ws, nb, stream)

    def engine(eng, T):
        items = [tuple(T[f"{k}.{i}"] for k in IN4) for i in range(len(sizes))]
        outs = eng.forward_ragged(items, tile=(th, tw), mode=spec["mode"], max_pass_pixels=mpp)
        return {f"out.{i}": o for i, o in enumerate(outs)}
    return Plan(bufs, issue, engine)


# ---- enhance family ------------------------------------------------------------------------------------------------
def build_enhance(spec, fn="wn_enhance_u8"):
    n, h, w = spec["shape"]
    f32 = spec.get("f32", True)
    npeers = spec.get("peers", 0)
    bufs = [_u8_in("rgb", (n, h, w, 3), h * w), _out("out_u8", "u8", (n, h, w, 3))]
    if f32:
        bufs.append(_out("out_f32", "f32", (n, 3, h, w)))
    bufs += [_out(f"peer.{k}", "u8", (n, h, w, 3)) for k in range(npeers)]
    mode = spec["mode"]

    def issue(P, ws, nb, stream, eng):
        L, hd = _lib(), _handle(eng)
        if fn == "wn_enhance_u8":
            return L.wn_enhance_u8(hd, P.ptr("rgb"), P.ptr("out_u8"), P.ptr("out_f32"), n, h, w, mode, ws, nb, stream)
        if fn == "wn_enhance_u8_peers":
            peers = _ptrs(P, [f"peer.{k}" for k in range(max(1, npeers))])
            return L.wn_enhance_u8_peers(hd, P.ptr("rgb"), P.ptr("out_u8"), P.ptr("out_f32"), peers, npeers, n, h, w,
                                         mode, ws, nb, stream)
        (th, tw), mpp = spec["tile"], spec["mpp"]
        return L.wn_enhance_u8_tiled(hd, P.ptr("rgb"), P.ptr("out_u8"), P.ptr("out_f32"), n, h, w, th, tw, mpp, mode,
                                     ws, nb, stream)

    def engine(eng, T):
        o32 = torch.empty((n, 3, h, w), device=T["rgb"].device) if f32 else None
        if fn == "wn_enhance_u8_tiled":
            u8 = eng.enhance_tiled(T["rgb"], tile=spec["tile"], mode=mode, out_f32=o32, max_pass_pixels=spec["mpp"])
        else:
            u8 = eng.enhance(T["rgb"], mode=mode, out_f32=o32)
        res = {"out_u8": u8, **{f"peer.{k}": u8 for k in range(npeers)}}
        if f32:
            res["out_f32"] = o32
        return res
    return Plan(bufs, issue, engine)


def build_enhance_ragged(spec):
    from waternet_b200 import _lib as L
    sizes, (th, tw), mpp = spec["sizes"], spec["tile"], spec["mpp"]
    f32 = spec.get("f32", [True] * len(sizes))
    bufs = [_u8_in(f"rgb.{i}", (h, w, 3), 7 * i + h, group="rgb") for i, (h, w) in enumerate(sizes)]
    bufs += [_out(f"out_u8.{i}", "u8", (h, w, 3), group="out_u8") for i, (h, w) in enumerate(sizes)]
    bufs += [_out(f"out_f32.{i}", "f32", (1, 3, h, w), group="out_f32") for i, (h, w) in enumerate(sizes) if f32[i]]

    def issue(P, ws, nb, stream, eng):
        table = (L.RaggedImage * len(sizes))(*[L.RaggedImage(P.ptr(f"rgb.{i}"), P.ptr(f"out_u8.{i}"),
                                                             P.ptr(f"out_f32.{i}"), h, w)
                                               for i, (h, w) in enumerate(sizes)])
        return _lib().wn_enhance_u8_ragged(_handle(eng), table, len(sizes), th, tw, mpp, spec["mode"], ws, nb, stream)

    def engine(eng, T):
        o32 = [torch.empty((1, 3, h, w), device="cuda") if f32[i] else None for i, (h, w) in enumerate(sizes)]
        u8 = eng.enhance_ragged([T[f"rgb.{i}"] for i in range(len(sizes))], tile=(th, tw), mode=spec["mode"],
                                out_f32=o32, max_pass_pixels=mpp)
        res = {f"out_u8.{i}": t for i, t in enumerate(u8)}
        res.update({f"out_f32.{i}": t for i, t in enumerate(o32) if t is not None})
        return res
    return Plan(bufs, issue, engine)


# ---- pre / post-processing -----------------------------------------------------------------------------------------
PRE_OUTS = ("x", "wb", "he", "gc", "wb_u8", "he_u8", "gc_u8")


def build_preprocess(spec):
    n, h, w = spec["shape"]
    want = spec.get("outs", PRE_OUTS)
    bufs = [_u8_in("rgb", (n, h, w, 3), h * w + 1)]
    bufs += [_out(k, "u8", (n, h, w, 3)) if k.endswith("_u8") else _out(k, "f32", (n, 3, h, w)) for k in want]

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_preprocess_u8(_handle(eng), P.ptr("rgb"), n, h, w, *[P.ptr(k) for k in PRE_OUTS], ws, nb,
                                       stream)

    def engine(eng, T):
        res = eng.preprocess(T["rgb"], tensors=True, images=True)
        return {k: res[k] for k in want}
    return Plan(bufs, issue, engine)


def build_white_balance_gray(spec):
    n, h, w = spec["shape"]
    bufs = [_u8_in("gray", (n, h, w), h * w + 2), _out("out", "u8", (n, h, w))]

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_white_balance_gray_u8(_handle(eng), P.ptr("gray"), P.ptr("out"), n, h, w, ws, nb, stream)
    return Plan(bufs, issue, lambda eng, T: {"out": eng.white_balance_gray(T["gray"])})


def build_resize(spec):
    sizes, (dh, dw), swap = spec["sizes"], spec["dst"], spec["swap"]
    n = len(sizes)
    bufs = [_u8_in(f"src.{i}", (h, w, 3), 3 * i + h, group="src") for i, (h, w) in enumerate(sizes)]
    bufs.append(_out("dst", "u8", (n, dh, dw, 3)))

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_resize_u8(_handle(eng), _ptrs(P, [f"src.{i}" for i in range(n)]),
                                   (c_int * n)(*[h for h, _ in sizes]), (c_int * n)(*[w for _, w in sizes]), n,
                                   P.ptr("dst"), dh, dw, swap, stream)
    return Plan(bufs, issue, lambda eng, T: {"dst": eng.resize_batch([T[f"src.{i}"] for i in range(n)], dh, dw,
                                                                     swap_rb=bool(swap))})


def build_postprocess(spec):
    n, h, w = spec["shape"]
    data = torch.rand((n, 3, h, w), generator=_gen(h * w)) * 1.4 - 0.2
    bufs = [Buf("in", "f32", (n, 3, h, w), "in", data), _out("out", "u8", (n, h, w, 3))]

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_postprocess_u8(_handle(eng), P.ptr("in"), P.ptr("out"), n, h, w, stream)
    return Plan(bufs, issue, lambda eng, T: {"out": eng.postprocess(T["in"])})


# ---- training ------------------------------------------------------------------------------------------------------
GIN4 = [f"gin.{k}" for k in range(4)]


def build_train(spec):
    n, h, w = spec["shape"]
    shape = (n, 3, h, w)
    bufs = _spec_ins(spec, shape)
    bufs += [_grad_in("grad_out", shape, 99), _out("out", "f32", shape)]
    bufs += _grads() + [_out(k, "f32", shape) for k in GIN4]

    def issue(P, ws, nb, stream, eng, stage="both"):
        L, hd = _lib(), _handle(eng)
        rc = 0
        if stage != "backward":
            rc = L.wn_forward_train(hd, *[P.ptr(k) for k in IN4], _st(P, IN4), P.ptr("out"), n, h, w, ws, nb, stream)
        if rc or stage == "forward":
            return rc
        return L.wn_backward(hd, P.ptr("grad_out"), _ptrs(P, GRADS), _ptrs(P, GIN4), n, h, w, ws, nb, stream)

    def engine(eng, T):
        out, saved = eng.forward_train(*[T[k] for k in IN4])
        grads, gin = eng.backward(T["grad_out"], saved, param_shapes(), want_input_grads=True)
        return {"out": out, **{f"grads.{i}": g for i, g in enumerate(grads)}, **dict(zip(GIN4, gin))}
    return Plan(bufs, issue, engine)


def build_train_ragged(spec):
    sizes = spec["sizes"]
    m = len(sizes)
    bufs = _ragged_ins(sizes, levels=spec.get("levels", False))
    bufs += [_grad_in(f"grad_out.{i}", (1, 3, h, w), 50 + i, group="grad_out") for i, (h, w) in enumerate(sizes)]
    bufs += [_out(f"out.{i}", "f32", (1, 3, h, w), group="out") for i, (h, w) in enumerate(sizes)]
    bufs += _grads()
    gin = [f"gin.{i}.{k}" for i in range(m) for k in range(4)]
    skip = set(spec.get("null_gin", ()))
    bufs += [_out(g, "f32", (1, 3) + sizes[int(g.split(".")[1])], group="gin") for g in gin if g not in skip]

    def issue(P, ws, nb, stream, eng, stage="both"):
        L, hd = _lib(), _handle(eng)
        hs, wss = (c_int * m)(*[h for h, _ in sizes]), (c_int * m)(*[w for _, w in sizes])
        rc = 0
        if stage != "backward":
            rc = L.wn_forward_train_ragged(hd, _ragged_tensors(P, sizes), m, ws, nb, stream)
        if rc or stage == "forward":
            return rc
        return L.wn_backward_ragged(hd, hs, wss, _ptrs(P, [f"grad_out.{i}" for i in range(m)]), _ptrs(P, GRADS),
                                    _ptrs(P, gin), m, ws, nb, stream)

    def engine(eng, T):
        items = [tuple(T[f"{k}.{i}"] for k in IN4) for i in range(m)]
        outs, saved = eng.forward_train_ragged(items)
        want = [[f"gin.{i}.{k}" not in skip for k in range(4)] for i in range(m)]
        grads, gins = eng.backward_ragged([T[f"grad_out.{i}"] for i in range(m)], saved, param_shapes(), want)
        res = {f"out.{i}": o for i, o in enumerate(outs)}
        if len(saved) == 1:  # Engine splits a batch with much padding into several calls: other fp32 sum orders
            res.update({f"grads.{i}": g for i, g in enumerate(grads)})
        res.update({f"gin.{i}.{k}": gins[i][k] for i in range(m) for k in range(4) if gins[i][k] is not None})
        return res
    return Plan(bufs, issue, engine)


def build_submodule_train(spec):
    """wn_confidence_maps_train -> _backward, or wn_refine_train -> _backward of ``which``.  ``spec["gin"]``: the
    input gradients asked for (the others are NULL: a non-NULL entry is a request).  ``spec["foreign"]``: the grads
    entries the stack does not own are given as NaN-filled guarded arenas instead of NULL; the call ignores them, so
    they must stay untouched."""
    n, h, w = spec["shape"]
    shape, stack, which = (n, 3, h, w), spec["stack"], spec.get("which", 0)
    cmg = stack == "cmg"
    names = IN4 if cmg else ("x", "xbar")
    gin_n = 4 if cmg else 2
    want_gin = spec.get("gin", (True,) * gin_n)
    bufs = _spec_ins(spec, shape, not cmg)
    bufs += [_grad_in("grad_out", shape, 98), _out("out", "f32", shape)] + _grads(stack, which)
    bufs += [_out(f"gin.{k}", "f32", shape) for k in range(gin_n) if want_gin[k]]
    foreign = []
    if spec.get("foreign"):
        shapes = param_shapes()
        foreign = [f"grads.{i}" for i in range(NUM_PARAMS) if i not in own_params(stack, which)]
        bufs += [Buf(g, "f32", shapes[int(g[6:])], "in", torch.full(shapes[int(g[6:])], float("nan")))
                 for g in foreign]

    def issue(P, ws, nb, stream, eng, stage="both"):
        L, hd = _lib(), _handle(eng)
        gin = _ptrs(P, [f"gin.{k}" for k in range(gin_n)]) if any(want_gin) or foreign else None
        rc = 0
        if cmg:
            if stage != "backward":
                rc = L.wn_confidence_maps_train(hd, *[P.ptr(k) for k in names], _st(P, names), P.ptr("out"), n, h, w,
                                                ws, nb, stream)
            if rc or stage == "forward":
                return rc
            return L.wn_confidence_maps_backward(hd, P.ptr("grad_out"), _ptrs(P, GRADS), gin, n, h, w, ws, nb, stream)
        if stage != "backward":
            rc = L.wn_refine_train(hd, which, P.ptr("x"), P.ptr("xbar"), _st(P, names), P.ptr("out"), n, h, w, ws, nb,
                                   stream)
        if rc or stage == "forward":
            return rc
        return L.wn_refine_backward(hd, which, P.ptr("grad_out"), _ptrs(P, GRADS), gin, n, h, w, ws, nb, stream)

    def engine(eng, T):
        own = list(own_params(stack, which))
        shapes = [param_shapes()[i] for i in own]
        if cmg:
            out, saved = eng.confidence_maps_train(*[T[k] for k in IN4])
            grads, gin = eng.confidence_maps_backward(T["grad_out"], saved, shapes, want_gin)
        else:
            out, saved = eng.refine_train(which, T["x"], T["xbar"])
            grads, gin = eng.refine_backward(which, T["grad_out"], saved, shapes, want_gin)
        res = {"out": out, **{f"grads.{i}": g for i, g in zip(own, grads)}}
        res.update({f"gin.{k}": t for k, t in enumerate(gin) if t is not None})
        return res
    return Plan(bufs, issue, engine)


def build_backward_tiled(spec):
    n, h, w = spec["shape"]
    shape, (th, tw), mpp = (n, 3, h, w), spec["tile"], spec["mpp"]
    stack, which = spec.get("stack", "all"), spec.get("which", 0)
    names = ("x", "xbar") if stack == "refiner" else IN4
    gin_n = len(names)
    bufs = _spec_ins(spec, shape, stack == "refiner")
    bufs += [_grad_in("grad_out", shape, 97)] + _grads(stack, which)
    bufs += [_out(f"gin.{k}", "f32", shape) for k in range(gin_n)]

    def issue(P, ws, nb, stream, eng):
        L, hd = _lib(), _handle(eng)
        common = (_st(P, names), P.ptr("grad_out"), _ptrs(P, GRADS), _ptrs(P, [f"gin.{k}" for k in range(gin_n)]),
                  n, h, w, th, tw, mpp, ws, nb, stream)
        if stack == "all":
            return L.wn_backward_tiled(hd, *[P.ptr(k) for k in IN4], *common)
        if stack == "cmg":
            return L.wn_confidence_maps_backward_tiled(hd, *[P.ptr(k) for k in IN4], *common)
        return L.wn_refine_backward_tiled(hd, which, P.ptr("x"), P.ptr("xbar"), *common)

    def engine(eng, T):
        own = list(own_params(stack, which))
        shapes = [param_shapes()[i] for i in own]
        kw = dict(tile=(th, tw), max_pass_pixels=mpp)
        if stack == "all":
            grads, gin = eng.backward_tiled(T["grad_out"], [T[k] for k in IN4], shapes, want_input_grads=True, **kw)
        elif stack == "cmg":
            grads, gin = eng.confidence_maps_backward_tiled(T["grad_out"], [T[k] for k in IN4], shapes,
                                                            want_inputs=(True,) * 4, **kw)
        else:
            grads, gin = eng.refine_backward_tiled(which, T["grad_out"], [T["x"], T["xbar"]], shapes,
                                                   want_inputs=(True, True), **kw)
        return {**{f"grads.{i}": g for i, g in zip(own, grads)}, **{f"gin.{k}": t for k, t in enumerate(gin)}}
    return Plan(bufs, issue, engine)


def build_backward_ragged_tiled(spec):
    sizes, (th, tw), mpp = spec["sizes"], spec["tile"], spec["mpp"]
    m = len(sizes)
    bufs = _ragged_ins(sizes, levels=spec.get("levels", False))
    bufs += [_grad_in(f"grad_out.{i}", (1, 3, h, w), 60 + i, group="grad_out") for i, (h, w) in enumerate(sizes)]
    bufs += _grads()
    gin = [f"gin.{i}.{k}" for i in range(m) for k in range(4)]
    bufs += [_out(g, "f32", (1, 3) + sizes[int(g.split(".")[1])], group="gin") for g in gin]

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_backward_ragged_tiled(_handle(eng), _ragged_tensors(P, sizes, out=False),
                                               _ptrs(P, [f"grad_out.{i}" for i in range(m)]), _ptrs(P, GRADS),
                                               _ptrs(P, gin), m, th, tw, mpp, ws, nb, stream)

    def engine(eng, T):
        items = [tuple(T[f"{k}.{i}"] for k in IN4) for i in range(m)]
        grads, gins = eng.backward_ragged_tiled([T[f"grad_out.{i}"] for i in range(m)], items, param_shapes(),
                                                tile=(th, tw), want_inputs=[[True] * 4] * m, max_pass_pixels=mpp)
        res = {f"grads.{i}": g for i, g in enumerate(grads)}
        res.update({f"gin.{i}.{k}": gins[i][k] for i in range(m) for k in range(4)})
        return res
    return Plan(bufs, issue, engine)


# ---- weights and the perceptual loss -------------------------------------------------------------------------------
def waternet_params():
    from oracle import forward as ofw
    sd = ofw.synthetic_state_dict(0, 3.0)
    return [sd[k].float() for k, _ in ofw.state_dict_spec()]


def vgg_params(seed=1234):
    g = _gen(seed)
    out = []
    for cin, cout in ((s[1], s[0]) for s in vgg_param_shapes()[0::2]):
        bound = (6.0 / (9 * cin)) ** 0.5
        out += [(torch.rand((cout, cin, 3, 3), generator=g) * 2 - 1) * bound, torch.rand((cout,), generator=g) * 0.1]
    return out


def build_pack(spec, vgg=False):
    params = vgg_params() if vgg else waternet_params()
    bufs = [Buf(f"params.{i}", "f32", tuple(p.shape), "in", p) for i, p in enumerate(params)]

    def issue(P, ws, nb, stream, eng):
        fn = _lib().wn_vgg_pack_weights if vgg else _lib().wn_pack_weights
        return fn(_handle(eng), _ptrs(P, [f"params.{i}" for i in range(len(params))]), stream)
    return Plan(bufs, issue, None)


def build_perceptual(spec):
    n, h, w = spec["shape"]
    shape, (th, tw), mpp = (n, 3, h, w), spec["tile"], spec["mpp"]
    bufs = [_f32_in("out", shape, 3), _f32_in("ref", shape, 4), _out("loss", "f32", (1,))]
    if spec.get("grad", True):
        bufs.append(_out("grad", "f32", shape))

    def issue(P, ws, nb, stream, eng):
        return _lib().wn_perceptual_loss(_handle(eng), P.ptr("out"), (c_int64 * 4)(*P.strides("out")), P.ptr("ref"),
                                         (c_int64 * 4)(*P.strides("ref")), n, h, w, th, tw, mpp, P.ptr("loss"),
                                         P.ptr("grad"), ws, nb, stream)

    def engine(eng, T):
        tile = None if th == 0 else (th, tw)
        loss, grad = eng.perceptual_loss(T["out"], T["ref"], tile=tile, want_grad=spec.get("grad", True),
                                         max_pass_pixels=mpp)
        res = {"loss": loss.reshape(1)}
        if grad is not None:
            res["grad"] = grad
        return res
    return Plan(bufs, issue, engine)


# ---- the table -----------------------------------------------------------------------------------------------------
def _nhw(spec):
    return spec["shape"]


def _shape_specs(shapes, modes, **extra):
    return [dict(shape=s, mode=m, **extra) for m in modes for s in shapes]


def _sizes_args(spec):
    return [h for h, _ in spec["sizes"]], [w for _, w in spec["sizes"]], len(spec["sizes"])


def _tiled_args(spec):
    return (*spec["shape"], *spec["tile"], spec["mpp"])


def _rejected_tiled(**extra):
    return [dict(shape=(2, 37, 53), tile=(23, 29), mpp=0, mode=FP32, **extra)]


TRAIN_SHAPES = [(1, 1, 1), (1, 24, 8), (1, 25, 17), (2, 37, 53), (300, 5, 7)]
TRAIN_RAGGED = [[(1, 1), (97, 118), (23, 7)], [(25, 9), (1, 1), (24, 17)]]
BWD_TILES = [((2, 37, 53), (23, 29)), ((1, 25, 17), (2, 13)), ((300, 5, 7), (2, 13))]
VGG_SPECS = [dict(shape=(1, 16, 16), tile=(0, 0), mpp=0), dict(shape=(1, 16, 16), tile=(32, 32), mpp=0, grad=False),
             dict(shape=(1, 17, 31), tile=(32, 32), mpp=0), dict(shape=(2, 40, 72), tile=(32, 32), mpp=0),
             dict(shape=(2, 40, 72), tile=(32, 32), mpp=160 * 176)]


def _bwd_specs(stack, whiches=(0,)):
    specs = []
    for k, (s, t) in enumerate(BWD_TILES):
        specs.append(dict(shape=s, tile=t, mpp=pass_pixels(*s, t), stack=stack, which=whiches[k % len(whiches)]))
    return specs


ROWS: List[Row] = [
    Row("forward", ("wn_forward",), "wn_forward_workspace_bytes", lambda s: (*_nhw(s), s["mode"]),
        IN4, ("out",), (), _shape_specs(EDGE, MODES) + [dict(shape=BIG, mode=DEFAULT)], build_forward),
    Row("confidence_maps", ("wn_confidence_maps",), "wn_submodule_workspace_bytes",
        lambda s: (*_nhw(s), s["mode"]), IN4, ("out",), (), _shape_specs(SUB_EDGE, MODES),
        lambda s: build_forward(s, "wn_confidence_maps")),
    Row("refine", ("wn_refine",), "wn_submodule_workspace_bytes", lambda s: (*_nhw(s), s["mode"]),
        ("x", "xbar"), ("out",), (),
        [dict(shape=sh, mode=m, which=k % 3) for m in MODES for k, sh in enumerate(SUB_EDGE)], build_refine),
    Row("forward_tiled", ("wn_forward_tiled",), "wn_forward_tiled_workspace_bytes",
        lambda s: (*_tiled_args(s), s["mode"]), IN4, ("out",), (), _tiled_specs(TC_MODES), build_forward_tiled,
        _rejected_tiled()),
    Row("confidence_maps_tiled", ("wn_confidence_maps_tiled",), "wn_submodule_tiled_workspace_bytes",
        lambda s: (*_tiled_args(s), s["mode"]), IN4, ("out",), (), _tiled_specs(TC_MODES, big=False)[::2],
        lambda s: build_forward_tiled(s, "wn_confidence_maps_tiled"), _rejected_tiled()),
    Row("refine_tiled", ("wn_refine_tiled",), "wn_submodule_tiled_workspace_bytes",
        lambda s: (*_tiled_args(s), s["mode"]), ("x", "xbar"), ("out",), (),
        [dict(sp, which=k % 3) for k, sp in enumerate(_tiled_specs(TC_MODES, big=False)[1::2])],
        lambda s: build_forward_tiled(s, "wn_refine_tiled"), _rejected_tiled(which=0)),
    Row("enhance_u8", ("wn_enhance_u8",), "wn_enhance_workspace_bytes", lambda s: (*_nhw(s), s["mode"]),
        ("rgb",), ("out_u8",), ("out_f32",),
        [dict(shape=sh, mode=m, f32=k % 2 == 0) for m in MODES for k, sh in enumerate(EDGE)]
        + [dict(shape=BIG, mode=DEFAULT, f32=True)], build_enhance),
    Row("enhance_u8_peers", ("wn_enhance_u8_peers",), "wn_enhance_workspace_bytes", lambda s: (*_nhw(s), s["mode"]),
        ("rgb",), ("out_u8", "peer"), ("out_f32",),
        [dict(shape=sh, mode=m, peers=2, f32=m != BF16X3) for m in MODES for sh in ((2, 33, 47), (1, 37, 53))],
        lambda s: build_enhance(s, "wn_enhance_u8_peers")),
    Row("enhance_u8_tiled", ("wn_enhance_u8_tiled",), "wn_enhance_tiled_workspace_bytes",
        lambda s: (*_tiled_args(s), s["mode"]), ("rgb",), ("out_u8",), ("out_f32",),
        [dict(sp, f32=k % 2 == 0) for k, sp in enumerate(_tiled_specs(TC_MODES))],
        lambda s: build_enhance(s, "wn_enhance_u8_tiled"), _rejected_tiled()),
    Row("enhance_u8_ragged", ("wn_enhance_u8_ragged",), "wn_enhance_ragged_workspace_bytes",
        lambda s: (*_sizes_args(s), *s["tile"], s["mpp"], s["mode"]), ("rgb",), ("out_u8",), ("out_f32",),
        [dict(sp, f32=[k % 2 == 0 for k in range(len(sp["sizes"]))]) for sp in _ragged_specs(TC_MODES)],
        build_enhance_ragged, [dict(sizes=RAGGED[0], tile=(37, 53), mpp=0, mode=FP32)]),
    Row("forward_ragged", ("wn_forward_ragged",), "wn_forward_ragged_workspace_bytes",
        lambda s: (*_sizes_args(s), *s["tile"], s["mpp"], s["mode"]), IN4, ("out",), (),
        _ragged_specs(TC_MODES), build_forward_ragged, [dict(sizes=RAGGED[0], tile=(37, 53), mpp=0, mode=FP32)]),
    Row("preprocess_u8", ("wn_preprocess_u8",), "wn_preprocess_workspace_bytes", _nhw, ("rgb",), (),
        PRE_OUTS, [dict(shape=s) for s in EDGE + [BIG]], build_preprocess),
    Row("white_balance_gray_u8", ("wn_white_balance_gray_u8",), "wn_white_balance_gray_workspace_bytes", _nhw,
        ("gray",), ("out",), (), [dict(shape=s) for s in EDGE + [BIG]], build_white_balance_gray),
    Row("resize_u8", ("wn_resize_u8",), None, None, ("src",), ("dst",), (),
        [dict(sizes=[(1, 1), (97, 118), (23, 7)], dst=(24, 17), swap=0),
         dict(sizes=[(97, 118), (1, 1)], dst=(1, 1), swap=1),
         dict(sizes=[(37, 53), (25, 9)], dst=(74, 106), swap=1),
         dict(sizes=[(1080, 1920)], dst=(540, 960), swap=0)], build_resize),
    Row("postprocess_u8", ("wn_postprocess_u8",), None, None, ("in",), ("out",), (),
        [dict(shape=s) for s in EDGE + [BIG]], build_postprocess),
    Row("train", ("wn_forward_train", "wn_backward"), "wn_train_workspace_bytes", _nhw,
        IN4 + ("grad_out",), ("out", "grads", "gin"), (), [dict(shape=s) for s in TRAIN_SHAPES], build_train),
    Row("train_ragged", ("wn_forward_train_ragged", "wn_backward_ragged"), "wn_train_ragged_workspace_bytes",
        lambda s: _sizes_args(s), IN4 + ("grad_out",), ("out", "grads", "gin"), (),
        [dict(sizes=s) for s in TRAIN_RAGGED]
        + [dict(sizes=TRAIN_RAGGED[0], null_gin=("gin.0.1", "gin.1.0", "gin.1.3"))],
        build_train_ragged),
    Row("confidence_maps_train", ("wn_confidence_maps_train", "wn_confidence_maps_backward"),
        "wn_submodule_train_workspace_bytes", lambda s: (*_nhw(s), 0), IN4 + ("grad_out",), ("out", "grads", "gin"),
        ("grads", "gin"), [dict(shape=s, stack="cmg") for s in TRAIN_SHAPES[:4]], build_submodule_train),
    Row("refine_train", ("wn_refine_train", "wn_refine_backward"), "wn_submodule_train_workspace_bytes",
        lambda s: (*_nhw(s), 1), ("x", "xbar", "grad_out"), ("out", "grads", "gin"), ("grads", "gin"),
        [dict(shape=s, stack="refiner", which=k) for k, s in enumerate(TRAIN_SHAPES[1:4])], build_submodule_train),
    Row("backward_tiled", ("wn_backward_tiled",), "wn_backward_tiled_workspace_bytes", _tiled_args,
        IN4 + ("grad_out",), ("grads", "gin"), (),
        _bwd_specs("all") + [dict(shape=BIG, tile=(998, 998), mpp=1 << 20, stack="all", which=0)],
        build_backward_tiled),
    Row("confidence_maps_backward_tiled", ("wn_confidence_maps_backward_tiled",),
        "wn_submodule_backward_tiled_workspace_bytes", lambda s: (*_tiled_args(s), 0), IN4 + ("grad_out",),
        ("grads", "gin"), ("grads",), _bwd_specs("cmg")[:2], build_backward_tiled),
    Row("refine_backward_tiled", ("wn_refine_backward_tiled",), "wn_submodule_backward_tiled_workspace_bytes",
        lambda s: (*_tiled_args(s), 1), ("x", "xbar", "grad_out"), ("grads", "gin"), ("grads",),
        _bwd_specs("refiner", (0, 1, 2)), build_backward_tiled),
    Row("backward_ragged_tiled", ("wn_backward_ragged_tiled",), "wn_backward_ragged_tiled_workspace_bytes",
        lambda s: (*_sizes_args(s), *s["tile"], s["mpp"]), IN4 + ("grad_out",), ("grads", "gin"), (),
        [dict(sizes=s, tile=t, mpp=ragged_pass_pixels(s, t)) for s, t in zip(TRAIN_RAGGED, ((23, 29), (2, 13)))],
        build_backward_ragged_tiled),
    Row("pack_weights", ("wn_pack_weights",), None, None, ("params",), (), (), [dict()], build_pack),
    Row("vgg_pack_weights", ("wn_vgg_pack_weights",), None, None, ("params",), (), (), [dict()],
        lambda s: build_pack(s, vgg=True)),
    Row("perceptual_loss", ("wn_perceptual_loss",), "wn_perceptual_loss_workspace_bytes",
        lambda s: (*_nhw(s), *s["tile"], s["mpp"]), ("out", "ref"), ("loss",), ("grad",), VGG_SPECS, build_perceptual),
]

ROW = {r.name: r for r in ROWS}

# Declared functions that take a workspace or write device memory and are not rows, with the reason.
EXCLUDED = {
    "wn_debug_forward_layer": "test aid",
    "wn_debug_backward_layer": "test aid",
    "wn_debug_vgg_layer": "test aid",
    "wn_peer_alloc": "cross-process IPC",
    "wn_peer_open": "cross-process IPC",
    "wn_peer_close": "cross-process IPC",
    "wn_peer_free": "cross-process IPC",
    "wn_memcpy_async": "a plain cudaMemcpyAsync of the caller's byte count",
    "wn_stream_write_value32": "a driver stream operation on one caller-given word",
    "wn_stream_wait_value32": "a driver stream operation that reads one caller-given word",
    "wn_build_tables_host": "host memory only",
    "wn_read_timings": "host memory only",
}


def header_functions(text: str) -> Dict[str, List[str]]:
    """The functions ``text`` (a C header) declares, each with its parameter declarations."""
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"#.*", "", text)
    out = {}
    for m in re.finditer(r"\b(wn_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text):
        out[m.group(1)] = [p.strip() for p in m.group(2).split(",") if p.strip() not in ("", "void")]
    return out


def writes_device_memory(params: List[str]) -> bool:
    """True when a parameter list has a workspace (``workspace``, ``ws``, ``train_workspace``) or a pointer to
    non-const data other than the handle and the stream."""
    for p in params:
        name = re.findall(r"\w+", p)[-1]
        if name in ("workspace", "ws", "train_workspace"):
            return True
        if "*" not in p or name in ("stream", "h") or p.startswith("wn_handle") or p.startswith("const wn_handle"):
            continue
        pointee = p[:p.index("*")].split()
        if "const" not in pointee:
            return True
    return False
