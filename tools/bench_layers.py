"""Per-launch times of the tensor-core forward in bench.py's resident step, set against the weight stream; one JSON line.

    python tools/bench_layers.py [--steps 30] [--warmup 5] [--mode default] [--mw1] [--tile C2=1x2 ...]

The step is bench.py's: 16 x 1920x1080 uint8 frames resident on the device through Engine.enhance, random-init
weights.  With wn_enable_timing on, each of the ten convolution launches is timed with CUDA events.  For each launch
this prints ms per step, TFLOP/s of the model's multiply-adds, and the GB/s of the weight stages the CTAs bulk-copy
from L2: every CTA work item copies every weight stage of its column group, so the bytes follow from the shapes and
the tile geometry, (8 mw) x (8 wgs) pixels per CTA tile (LAYERS below, the spec table of csrc/conv_umma.cu; --mw1
computes them for 8 x 16-pixel tiles everywhere, the geometry before 16 x 16 tiles; --tile NAME=MWxWGS sets one
launch's mw and wgs, to describe a library built from another table).  One L2 read-bandwidth proxy is printed beside them: repeated sums
over a 16 MB fp32 tensor that stays resident in the 50 MB L2.  The card's name and power limit are in the same JSON.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# launch: (timing slot, ks, cinpad, npad per block, nblk, mw, ng, wgs, model multiply-adds per pixel)
LAYERS = {
    "L1": (0, 7, 16, 224, 1, 1, 1, 2, 75264 + 3 * 9408),
    "C2": (1, 5, 128, 128, 1, 1, 1, 3, 409600),
    "C3": (2, 3, 128, 128, 1, 1, 1, 3, 147456),
    "C4": (3, 1, 128, 64, 1, 1, 1, 3, 8192),
    "C5": (4, 7, 64, 64, 1, 2, 1, 2, 200704),
    "C6": (5, 5, 64, 64, 1, 2, 1, 3, 102400),
    "C7": (6, 3, 64, 64, 1, 2, 1, 3, 36864),
    "C8": (7, 3, 64, 16, 1, 1, 1, 3, 1728),
    "R2": (9, 5, 96, 32, 3, 1, 1, 3, 3 * 25600),
    "R3": (10, 3, 96, 16, 1, 1, 1, 3, 3 * 864),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers stay valid, only unlabelled
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e.__class__.__name__})"}


def weight_bytes_per_image(h, w, ks, cinpad, npad, mw, wgs):
    """Weight-stage bytes all CTAs of one launch copy for one image: per (8 mw x 8 wgs)-pixel tile, 64 B per output
    channel per (16-channel chunk, tap) -- the same for every column group split of the npad channels."""
    tiles = -(-w // (8 * mw)) * -(-h // (8 * wgs))
    return tiles * (cinpad // 16) * ks * ks * npad * 64


def l2_proxy_gbs(reps=200):
    """Read GB/s of torch.sum over a 16 MB fp32 tensor that stays in L2 (a proxy: one kernel, one access pattern)."""
    x = torch.rand(4 << 20, device="cuda")
    out = torch.empty((), device="cuda")
    for _ in range(20):
        torch.sum(x, dim=0, out=out)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        torch.sum(x, dim=0, out=out)
    b.record()
    b.synchronize()
    return x.numel() * 4 * reps / (a.elapsed_time(b) * 1e-3) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--mode", choices=["default", "bf16x3", "bf16_fp8"], default="default")
    ap.add_argument("--mw1", action="store_true", help="weight bytes for 8 x 16-pixel tiles in every layer")
    ap.add_argument("--tile", action="append", default=[], metavar="NAME=MWxWGS",
                    help="the tile of one launch in the library measured, e.g. C2=1x2")
    args = ap.parse_args()
    geometry = {name: (1, 2) if args.mw1 else (spec[5], spec[7]) for name, spec in LAYERS.items()}
    for t in args.tile:
        name, mw_wgs = t.split("=")
        geometry[name] = tuple(int(v) for v in mw_wgs.split("x"))
    if not torch.cuda.is_available():
        raise SystemExit("bench_layers.py needs a CUDA device (H100)")
    from bench import bench_state_dict, synthetic_batch
    from waternet_b200.api import Enhancer
    from waternet_b200.net import WaterNet

    model = WaterNet(precision=args.mode)
    model.load_state_dict(bench_state_dict(), strict=True)
    model = model.cuda().eval()
    eng = Enhancer(model, device=torch.device("cuda", 0)).engine
    mode = model._mode()
    B, H, W = args.batch, args.height, args.width
    dev_in = torch.from_numpy(synthetic_batch(B, H, W, seed=0)).cuda()
    dev_out = torch.empty_like(dev_in)
    nb = eng.chunk_images(B, H, W)

    def step():
        for a in range(0, B, nb):
            eng.enhance(dev_in[a:a + nb], mode=mode, out_u8=dev_out[a:a + nb])

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    eng.enable_timing(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    ms, cnt = eng.read_timings()
    eng.enable_timing(False)
    step_ms = e0.elapsed_time(e1) / args.steps
    l2 = l2_proxy_gbs()

    layers = {}
    for name, (slot, ks, cinpad, npad, nblk, _, ng, _, macs) in LAYERS.items():
        if not cnt[slot]:
            continue
        t = ms[slot] / args.steps
        wbytes = B * weight_bytes_per_image(H, W, ks, cinpad, npad, *geometry[name])
        layers[name] = {"ms_per_step": round(t, 3), "tflops": round(2.0 * macs * H * W * B / (t * 1e-3) / 1e12, 1),
                        "weight_bytes_per_px": round(wbytes / (B * H * W)),
                        "weight_stream_gbs": round(wbytes / (t * 1e-3) / 1e9)}
    total_w = sum(B * weight_bytes_per_image(H, W, *LAYERS[k][1:4], *geometry[k]) for k in layers)
    print(json.dumps({"metric": "tensor_core_launches", **card(), "mode": args.mode,
                      "workload": f"{B} x {W}x{H} resident (bench.py step)", "steps": args.steps,
                      "geometry": {k: f"{8 * mw}x{8 * wgs}" for k, (mw, wgs) in geometry.items()},
                      "ms_per_step": round(step_ms, 3), "images_per_s": round(B / (step_ms * 1e-3), 2),
                      "conv_ms_per_step": round(sum(v["ms_per_step"] for v in layers.values()), 3),
                      "weight_stream_gbs_step_avg": round(total_w / (step_ms * 1e-3) / 1e9),
                      "l2_read_proxy_gbs": round(l2), "layers": layers}))


if __name__ == "__main__":
    main()
