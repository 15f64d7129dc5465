"""A training step over images of their own sizes: one ragged step against the per-image loop; prints one JSON line.

    python tools/bench_ragged_train.py [--rounds 5] [--warmup 2] [--seed 0]

A step is forward, MSE against a random target and backward with the 34 parameter gradients (no VGG loss, no
optimizer), over a seeded mix of 32 sizes from 64 x 64 to 512 x 384 (--max-size H W for another upper end).  Paths, alternated over --rounds:
  ragged     Engine.forward_train_ragged / backward_ragged (wn_forward_train_ragged / wn_backward_ragged)
  per_image  Engine.forward_train / backward of each image, the parameter gradients accumulated
Reported: median ms per step, peak device memory of one step, kernel launches of one step, and the plan (training
calls, slot pixels over image pixels).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import random
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_tiled import card  # noqa: E402
from bench_tiled_train import peak_step_bytes, timed_step_ms  # noqa: E402


def sizes_mix(seed, n=32, lo=64, hi=(512, 384)):
    rng = random.Random(seed)
    return [(rng.randrange(lo, hi[0] + 1, 8), rng.randrange(lo, hi[1] + 1, 8)) for _ in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-size", type=int, nargs=2, default=(512, 384), metavar=("H", "W"),
                    help="the largest height and width of the mix (smallest 64 x 64)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged_train.py needs a CUDA device (H100)")
    from waternet_b200.engine import ragged_train_calls
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet().cuda().train()
    eng = model.engine()
    shapes = [p.shape for p in model.parameters()]
    sizes = sizes_mix(args.seed, hi=tuple(args.max_size))
    gen = torch.Generator(device="cuda").manual_seed(args.seed)
    items = [tuple(torch.rand(1, 3, h, w, device="cuda", generator=gen) for _ in range(4)) for h, w in sizes]
    targets = [torch.rand(1, 3, h, w, device="cuda", generator=gen) for h, w in sizes]
    total_px = sum(h * w for h, w in sizes)

    def mse_grad(out, t):  # d(mean over images of mse_i)/d(out)
        return 2 * (out - t) / (out.numel() * len(sizes))

    def ragged():
        outs, saved = eng.forward_train_ragged(items)
        eng.backward_ragged([mse_grad(o, t) for o, t in zip(outs, targets)], saved, shapes)

    def per_image():
        acc = None
        for it, t in zip(items, targets):
            out, saved = eng.forward_train(*it)
            g = eng.backward(mse_grad(out, t), saved, shapes)
            acc = g if acc is None else torch._foreach_add(acc, g)

    paths = {"ragged": ragged, "per_image": per_image}
    for _ in range(args.warmup):
        for fn in paths.values():
            fn()
    times = {k: [] for k in paths}
    for _ in range(args.rounds):
        for k, fn in paths.items():
            times[k].append(timed_step_ms(fn))
    calls = ragged_train_calls(sizes, eng.TRAIN_MAX_PIXELS)
    slot_px = 0
    for c in calls:
        sub = [sizes[i] for i in c]
        slot_px += len(c) * max(h for h, _ in sub) * max(w for _, w in sub)
    res = {"metric": "ragged_training_step", **card(), "rounds": args.rounds, "images": len(sizes),
           "image_pixels": total_px, "training_calls": len(calls), "slot_pixels_over_image_pixels":
           round(slot_px / total_px, 3), "step": "forward + mse + backward (34 parameter gradients), no VGG"}
    for k, fn in paths.items():
        torch.cuda.empty_cache()
        before = eng.launch_count
        fn()
        torch.cuda.synchronize()
        launches = eng.launch_count - before
        res[k] = {"ms_per_step": round(statistics.median(times[k]), 2), "ms": [round(t, 2) for t in times[k]],
                  "peak_bytes": peak_step_bytes(fn), "launches": launches,
                  "mpx_per_s": round(total_px / 1e6 / (statistics.median(times[k]) / 1e3), 1)}
    res["ragged_vs_per_image"] = round(res["ragged"]["ms_per_step"] / res["per_image"]["ms_per_step"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
