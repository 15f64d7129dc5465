"""A ragged batch (images of mixed sizes) in one call against a per-image loop, on one GPU; prints one JSON line.

    python tools/bench_ragged.py [--rounds 3] [--warmup 2] [--mode default] [--images 100] [--tiles 998,2048]

A seeded directory-like mix of ~100 images, thumbnails to 1080p plus odd sizes, enhanced two ways:
- resident: a per-image Engine.enhance loop against one Engine.enhance_ragged call (device buffers; CUDA events);
- host buffers: a per-image Enhancer loop (inference.py without --batch) against one Enhancer.enhance_many call
  (numpy in, numpy out; wall clock, copies included).
The ragged side runs once per --tiles entry: 998 (Engine.DEFAULT_TILE, what enhance_many uses without a tile) cuts
the 1080p frames into four windows; 2048 keeps every image of the mix whole.  Rounds alternate between the two sides
of each comparison after a warm-up of both.  Reported: images/s and Mpx/s,
the padding fraction and recompute factor of the plan, the wn_launch_count delta of each side, and whether the
outputs are bitwise equal.  The card's name and power limit are read with an nvidia-smi query; they belong beside
every number this prints.
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_tiled import card, frames, timed  # noqa: E402

COMMON = [(112, 112), (240, 320), (300, 400), (480, 640), (533, 800), (720, 1280), (1080, 1920)]
ODD = [(37, 53), (113, 117), (77, 141), (250, 333)]


def mix(n, seed):
    rng = random.Random(seed)
    sizes = [rng.choice(ODD) if rng.random() < 0.2 else rng.choice(COMMON) for _ in range(n)]
    return [frames(1, h, w, seed * 1000 + i)[0] for i, (h, w) in enumerate(sizes)]


def plan_stats(sizes, tile):
    from waternet_b200.engine import ragged_plan
    passes = ragged_plan(sizes, *tile)
    slots = sum(len(p["windows"]) * p["slot"][0] * p["slot"][1] for p in passes)
    valid = sum(r["vh"] * r["vw"] for p in passes for r in p["windows"])
    return {"passes": len(passes), "windows": sum(len(p["windows"]) for p in passes),
            "padding_fraction": round(1 - valid / slots, 4),
            "recompute_factor": round(valid / sum(h * w for h, w in sizes), 4)}


def launches(eng, fn):
    before = eng.launch_count
    fn()
    torch.cuda.synchronize()
    return eng.launch_count - before


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--images", type=int, default=100)
    ap.add_argument("--tiles", type=str, default="998,2048")
    ap.add_argument("--mode", choices=["default", "bf16x3", "bf16_fp8"], default="default")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged.py needs a CUDA device (H100)")
    from waternet_b200.api import Enhancer
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet(precision=args.mode).cuda().eval()  # default init, as bench.py
    eng = model.engine()
    mode = model._mode()
    tiles = [int(t) for t in args.tiles.split(",")]
    imgs = mix(args.images, 0)
    sizes = [tuple(i.shape[:2]) for i in imgs]
    mpx = sum(h * w for h, w in sizes) / 1e6
    res = {"metric": "ragged_vs_per_image_enhance", **card(), "mode": args.mode, "images": len(imgs),
           "mpx": round(mpx, 2), "rounds": args.rounds}

    def compare(a, b, clock, n_a, n_b, same):
        """alternated rounds of a and b after a warm-up of both"""
        for _ in range(args.warmup):
            a()
            b()
        t_a, t_b = [], []
        for _ in range(args.rounds):
            t_a.append(clock(a))
            t_b.append(clock(b))
        ma, mb = statistics.median(t_a), statistics.median(t_b)
        return {f"{n_a}_images_s": round(len(imgs) / ma, 1), f"{n_b}_images_s": round(len(imgs) / mb, 1),
                f"{n_a}_mpx_s": round(mpx / ma, 1), f"{n_b}_mpx_s": round(mpx / mb, 1), "speedup": round(ma / mb, 3),
                f"{n_a}_s": [round(t, 4) for t in t_a], f"{n_b}_s": [round(t, 4) for t in t_b],
                f"{n_a}_launches": launches(eng, a), f"{n_b}_launches": launches(eng, b), "bitwise_equal": same()}

    def wall(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        return time.perf_counter() - t0

    # ---- resident: device buffers in and out
    out_a = [torch.empty_like(i) for i in imgs]
    out_b = [torch.empty_like(i) for i in imgs]
    loop = lambda: [eng.enhance(i[None], mode=mode, out_u8=o[None]) for i, o in zip(imgs, out_a)]  # noqa: E731
    for tile in tiles:
        ragged = lambda: eng.enhance_ragged(imgs, tile=tile, mode=mode, out_u8=out_b)  # noqa: E731
        r = compare(loop, ragged, timed, "per_image", "ragged",
                    lambda: all(torch.equal(a, b) for a, b in zip(out_a, out_b)))
        res[f"resident_tile_{tile}"] = {**plan_stats(sizes, (tile, tile)), **r,
                                        "ragged_workspace_bytes": eng.ragged_workspace_bytes(sizes, tile, mode)}
        for o in out_b:
            o.zero_()

    # ---- host buffers: numpy in, numpy out (the per-image Enhancer is today's inference.py)
    arrs = [i.cpu().numpy() for i in imgs]
    got = {}
    per = Enhancer(model)

    def per_image():
        got["a"] = [per(a) for a in arrs]

    for tile in tiles:
        enh = Enhancer(model, tile=tile)

        def many():
            got["b"] = enh.enhance_many(arrs)

        res[f"host_buffers_tile_{tile}"] = compare(
            per_image, many, wall, "per_image", "enhance_many",
            lambda: all(np.array_equal(a, b) for a, b in zip(got["a"], got["b"])))
    res["f8_overflowed"] = eng.f8_overflowed()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
