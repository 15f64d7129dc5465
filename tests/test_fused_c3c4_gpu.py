"""cmg.conv4 computed in cmg.conv3's epilogue (UmmaCfg kFmtFuse1x1): one launch instead of two in every inference
pass.  The fused launch feeds cmg.conv4 the bits cmg.conv3's own epilogue would have stored and issues, per output
column, the products of cmg.conv4's own launch in the same order, so the product library and the WN_UMMA_UNFUSED_C4
library (cmg.conv4 as a launch of its own) must give bitwise-equal fp32 and uint8 outputs in both tensor-core modes:
whole images (1080p, and partial 8 x 24 tiles), a tiled and a ragged enhance, fp32 tensors through WaterNet.forward and
forward_many, and a batch whose activations leave the e4m3 range, so that the conditional bf16x3 chain runs fused too.
The fixture builds the WN_UMMA_UNFUSED_C4 library next to the product library when it is missing."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
PKG = os.path.join(ROOT, "waternet_b200")
PRODUCT_LIB = os.path.join(PKG, "libwaternet_b200.so")
UNFUSED_LIB_NAME = "libwaternet_b200_unfused_c4.so"


@pytest.fixture(scope="module")
def unfused_lib():
    sys.path.insert(0, ROOT)
    from waternet_b200 import build
    return build.build(defines=("WN_UMMA_UNFUSED_C4",), lib_name=UNFUSED_LIB_NAME)


# run in a process of its own per library: the binding loads one library per process (WATERNET_B200_LIB)
_DUMP = r"""
import sys, torch
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import forward_reference as fr
from oracle import forward as ofw
from waternet_b200.net import WaterNet

def model(precision, sd):
    m = WaterNet(precision=precision)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()

def frames(sizes, seed):
    return [torch.from_numpy(ofw.synthetic_image(seed + i, h, w, "smooth" if i % 2 else "noise")).cuda()
            for i, (h, w) in enumerate(sizes)]

out = {}
for mode in ("bf16x3", "bf16_fp8"):
    m = model(mode, ofw.synthetic_state_dict(11, 3.0))
    eng, md = m.engine(), m._mode()
    for n, h, w in ((2, 1080, 1920), (1, 37, 53), (3, 113, 117)):
        x = torch.stack(frames([(h, w)] * n, h + w))
        f32 = torch.full((n, 3, h, w), float("nan"), device="cuda")
        before = eng.launch_count
        out[(mode, "enhance_u8", n, h, w)] = eng.enhance(x, mode=md, out_f32=f32).cpu()
        torch.cuda.synchronize()
        out[(mode, "enhance_launches", n, h, w)] = eng.launch_count - before
        out[(mode, "enhance_f32", n, h, w)] = f32.cpu()
        res = eng.preprocess(x, tensors=True)
        with torch.no_grad():
            out[(mode, "forward_levels", n, h, w)] = m(*[res[k] for k in ("x", "wb", "he", "gc")]).cpu()
            if h < 1080:  # random floats: the first layer's bf16x3 form
                ins = [t.cuda() for t in fr.make_inputs("floats", n, h, w, h * 1000 + w)]
                out[(mode, "forward_floats", n, h, w)] = m(*ins).cpu()
        torch.cuda.synchronize()
        out[(mode, "overflowed", n, h, w)] = eng.f8_overflowed()
    x = torch.stack(frames([(121, 203)] * 2, 5))
    f32 = torch.full((2, 3, 121, 203), float("nan"), device="cuda")
    out[(mode, "tiled_u8")] = eng.enhance_tiled(x, tile=(37, 53), mode=md, out_f32=f32, max_pass_pixels=20_000).cpu()
    out[(mode, "tiled_f32")] = f32.cpu()
    sizes = [(1, 1), (23, 7), (25, 9), (49, 40), (71, 53), (97, 118)]
    images = frames(sizes, 70)
    f32s = [torch.full((1, 3, h, w), float("nan"), device="cuda") for h, w in sizes]
    got = eng.enhance_ragged(images, tile=(43, 61), mode=md, out_f32=f32s, max_pass_pixels=30_000)
    for i in range(len(sizes)):
        out[(mode, "ragged_u8", i)] = got[i].cpu()
        out[(mode, "ragged_f32", i)] = f32s[i].cpu()
    ins = [[t.cuda() for t in fr.make_inputs("floats", 1, h, w, 7 * h + w)] for h, w in sizes[1:]]
    with torch.no_grad():
        many = m.forward_many(*[[i[k] for i in ins] for k in range(4)])
    for i, t in enumerate(many):
        out[(mode, "forward_many", i)] = t.cpu()
    torch.cuda.synchronize()
    out[(mode, "overflowed")] = eng.f8_overflowed()

# refiner activations beyond the e4m3 range: the fp8-correction pass raises the flag and the conditional bf16x3 chain
# recomputes the batch within the call (both chains run cmg.conv3 and cmg.conv4 as one launch)
sd = ofw.synthetic_state_dict(0, 3.0)
sd["wb_refiner.conv1.weight"] = sd["wb_refiner.conv1.weight"] * 400.0
sd["wb_refiner.conv2.weight"] = sd["wb_refiner.conv2.weight"] / 400.0
m = model("default", sd)
x = torch.stack(frames([(40, 56)] * 3, 5))
f32 = torch.full((3, 3, 40, 56), float("nan"), device="cuda")
out[("overflow", "enhance_u8")] = m.engine().enhance(x, mode=m._mode(), out_f32=f32).cpu()
out[("overflow", "enhance_f32")] = f32.cpu()
torch.cuda.synchronize()
out[("overflow", "overflowed")] = m.engine().f8_overflowed()
torch.save(out, sys.argv[3])
"""


def _dump(lib, path):
    env = dict(os.environ, WATERNET_B200_LIB=lib)
    res = subprocess.run([sys.executable, "-c", _DUMP, ROOT, TESTS, path], env=env, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-4000:]
    return torch.load(path)


def test_fused_conv3_conv4_bitwise_equal_to_two_launches(unfused_lib, tmp_path):
    prod = _dump(PRODUCT_LIB, str(tmp_path / "product.pt"))
    ref = _dump(unfused_lib, str(tmp_path / "unfused.pt"))
    assert prod.keys() == ref.keys()
    for k in ref:
        if "enhance_launches" in k:
            continue
        if isinstance(ref[k], torch.Tensor):
            assert torch.equal(prod[k], ref[k]), k
        else:
            assert prod[k] == ref[k], k
    # the 1080p case ran in the fp8-correction mode, and the range-guard case took the bf16x3 chain
    assert not ref[("bf16_fp8", "overflowed", 2, 1080, 1920)]
    assert ref[("overflow", "overflowed")]
    # one launch fewer per chain and pass: the bf16x3 mode runs one chain, the fp8-correction mode two (the
    # conditional bf16x3 chain is enqueued behind it)
    case = (2, 1080, 1920)
    assert ref[("bf16x3", "enhance_launches") + case] - prod[("bf16x3", "enhance_launches") + case] == 1
    assert ref[("bf16_fp8", "enhance_launches") + case] - prod[("bf16_fp8", "enhance_launches") + case] == 2
