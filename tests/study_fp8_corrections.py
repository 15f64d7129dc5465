"""CPU emulation of the tensor-core operand schemes (test infrastructure; imports the oracle).

How much accuracy the forward keeps when the two bf16 correction passes of the bf16x3 scheme
(a_lo x w, a_hi x w_lo) are evaluated with fp8 operands instead -- e4m3 (or e5m2) activations x e4m3
weights with a static per-layer power-of-two scale -- as the library's WN_MODE_BF16_FP8 does with one
e4m3 wgmma (waternet_b200/csrc/umma_conv.cuh, UmmaCfg FMT).  Everything is evaluated in
float64 except the operand roundings, so the numbers isolate the quantisation error.

    python tests/study_fp8_corrections.py        # prints the table quoted in DESIGN.md section 4.2 / 9

tests/test_fp8_scheme_cpu.py runs a small case of it as a regression test.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.nn.functional as F

from oracle import forward as ofw
from oracle import preprocess as opre

# the layers the library runs with the fp8 correction pass (conv_umma.cu: the f8 column of kSpecs)
LIBRARY_F8_LAYERS = {"cmg.conv2", "cmg.conv3", "cmg.conv5", "cmg.conv6", "cmg.conv7",
                     "wb_refiner.conv2", "ce_refiner.conv2", "gc_refiner.conv2"}


def _bf16(x):
    return x.to(torch.bfloat16).to(torch.float64)


def _q8(x, dt):
    return x.to(torch.float32).to(dt).to(torch.float64)


def conv_scheme(a, w, b, k, scheme):
    """One "same" convolution with the operand roundings of `scheme`:
    exact | bf16x1 | 2pass (a_lo x w dropped) | bf16x3 | fp8_<fmt> (a_lo x w in fp8) | fp8x2_<fmt> (both corrections)."""
    a, w, b = a.double(), w.double(), b.double()
    pad = k // 2
    if scheme == "exact":
        return F.conv2d(a, w, b, padding=pad)
    a_hi = _bf16(a)
    a_lo = _bf16(a - a_hi)
    w_hi = _bf16(w)
    w_lo = _bf16(w - w_hi)
    out = F.conv2d(a_hi, w_hi, None, padding=pad)
    if scheme == "bf16x1":
        return out + b.view(1, -1, 1, 1)
    if scheme.startswith("fp8"):
        adt = {"e5m2": torch.float8_e5m2, "e4m3": torch.float8_e4m3fn}[scheme.split("_")[1]]
        ws = 2.0 ** np.floor(np.log2(224.0 / max(w.abs().max().item(), 1e-30)))  # max|w| lands in [112, 224]
        out = out + F.conv2d(_q8((a - a_hi) * 512.0, adt) / 512.0, _q8(w * ws, torch.float8_e4m3fn) / ws, None,
                             padding=pad)
        if scheme.startswith("fp8x2"):
            out = out + F.conv2d(_q8(a, adt), _q8(w_lo * ws * 512.0, torch.float8_e4m3fn) / (ws * 512.0), None,
                                 padding=pad)
        else:
            out = out + F.conv2d(a_hi, w_lo, None, padding=pad)
        return out + b.view(1, -1, 1, 1)
    out = out + F.conv2d(a_hi, w_lo, None, padding=pad)
    if scheme == "bf16x3":
        out = out + F.conv2d(a_lo, w_hi, None, padding=pad)
    return out + b.view(1, -1, 1, 1)


def forward(sd, x, wb, he, gc, scheme, f8_layers=None):
    """WaterNet forward (net.py:45-56, 75-80, 99-108) with `scheme` in the layers of `f8_layers`
    (None = every layer) and bf16x3 in the others ("exact" applies everywhere)."""
    def conv(prefix, t, k):
        s = scheme if (scheme == "exact" or f8_layers is None or prefix in f8_layers) else "bf16x3"
        return conv_scheme(t, sd[prefix + ".weight"], sd[prefix + ".bias"], k, s)

    t = torch.cat([x, wb, he, gc], 1).double()
    for name, _, _, k in ofw.CMG_LAYERS[:-1]:
        t = F.relu(conv(f"cmg.{name}", t, k))
    cm = torch.sigmoid(conv("cmg.conv8", t, 3))
    out = 0
    for r, (ref, other) in enumerate(zip(ofw.REFINERS, (wb, he, gc))):
        u = torch.cat([x, other], 1).double()
        for name, _, _, k in ofw.REFINER_LAYERS:
            u = F.relu(conv(f"{ref}.{name}", u, k))
        out = out + u * cm[:, r:r + 1]
    return out


def inputs(seed, size, kind):
    rgb = ofw.synthetic_image(seed, size, size, kind)
    wbi, gci, hei = opre.transform(rgb)
    ten = lambda a: torch.from_numpy(a.astype(np.float32) / 255).permute(2, 0, 1)[None]
    return [ten(rgb), ten(wbi), ten(hei), ten(gci)]


def rel_err(out, ref):
    return ((out - ref).abs().max() / ref.abs().max()).item()


if __name__ == "__main__":
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    for gain in (1.0, 3.0):
        for seed in (0, 1):
            sd = ofw.synthetic_state_dict(seed, gain)
            ins = inputs(seed + 10, 96, "smooth" if seed == 0 else "noise")
            ref = forward(sd, *ins, "exact")
            res = {s: rel_err(forward(sd, *ins, s), ref)
                   for s in ("bf16x3", "fp8_e5m2", "fp8x2_e5m2", "fp8x2_e4m3", "2pass", "bf16x1")}
            res["library(fp8x2_e4m3 in its 6 layers)"] = rel_err(forward(sd, *ins, "fp8x2_e4m3", LIBRARY_F8_LAYERS), ref)
            print("gain", gain, "seed", seed, " ".join(f"{k}={v:.2e}" for k, v in res.items()), flush=True)
