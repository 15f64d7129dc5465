"""A windowed training step over images of their own sizes: WaterNet.forward_many under grad_tile against the
per-item windowed loop it replaces; prints one JSON line.

    python tools/bench_ragged_tiled_train.py [--rounds 3] [--warmup 1] [--seed 0] [--tile 998]

A step is forward, MSE against a random target and backward, with the 34 parameter gradients and the input
gradients (no VGG loss, no optimizer).  Arms, alternated over --rounds after --warmup steps of each:
  ragged_tiled  WaterNet.forward_many with grad_tile (wn_forward_ragged + wn_backward_ragged_tiled: one call each)
  per_item      model(*item) per item with grad_tile (wn_forward_tiled + wn_backward_tiled per item)
  untiled       WaterNet.forward_many without grad_tile (the ragged training step), where its activations fit
Workloads: the two mixes of bench_ragged_train.py (32 images of 64-160 pixels per side; 32 of 64 x 64 to
512 x 384), and 16 photo sizes up to 1080p plus one 3000 x 4000 image, which the untiled step cannot hold.
Reported per arm: median ms per step, Mpx/s, peak device memory and kernel launches of one step; per workload the
plan (windows, passes, slot pixels over window pixels) and whether the outputs and input gradients of ragged_tiled
and per_item are equal bit for bit.  The card's name and power limit are read in the same run.
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

from bench_ragged_train import sizes_mix  # noqa: E402
from bench_tiled import card  # noqa: E402
from bench_tiled_train import peak_step_bytes, timed_step_ms  # noqa: E402

PHOTO_SIZES = [(1080, 1920), (1920, 1080), (720, 1280), (1280, 720), (768, 1024), (1024, 768), (600, 800),
               (480, 640), (1080, 1440), (900, 1200)]


def workloads(seed):
    rng = random.Random(seed)
    return {"small_64_160": sizes_mix(seed, hi=(160, 160)),
            "mixed_64_512x384": sizes_mix(seed, hi=(512, 384)),
            "photos_1080p_and_12mpx": [rng.choice(PHOTO_SIZES) for _ in range(16)] + [(3000, 4000)]}


def run(model, sizes, args):
    from waternet_b200.engine import TRAIN_PASS_PIXELS, ragged_plan
    eng = model.engine()
    gen = torch.Generator(device="cuda").manual_seed(args.seed)
    items = [tuple(torch.rand(1, 3, h, w, device="cuda", generator=gen).requires_grad_(True) for _ in range(4))
             for h, w in sizes]
    targets = [torch.rand(1, 3, h, w, device="cuda", generator=gen) for h, w in sizes]
    leaves = [t for it in items for t in it]
    total_px = sum(h * w for h, w in sizes)

    def step(outs_of):
        model.zero_grad(set_to_none=True)
        for t in leaves:
            t.grad = None
        outs = outs_of()
        loss = sum(torch.nn.functional.mse_loss(o, t) for o, t in zip(outs, targets)) / len(sizes)
        loss.backward()
        return outs

    def ragged(tile):
        def fn():
            model.grad_tile = tile
            return step(lambda: model.forward_many(*[list(t) for t in zip(*items)]))
        return fn

    def per_item():
        model.grad_tile = args.tile
        return step(lambda: [model(*it) for it in items])

    arms = {"ragged_tiled": ragged(args.tile), "per_item": per_item}
    untiled_bytes = total_px * 5616  # kTrainBytesPerPixel, before slot padding
    if untiled_bytes < 0.5 * torch.cuda.get_device_properties(0).total_memory:
        arms["untiled"] = ragged(None)
    res = {"images": len(sizes), "image_pixels": total_px}
    passes = ragged_plan(sizes, args.tile, args.tile, TRAIN_PASS_PIXELS)
    win_px = sum(r["vh"] * r["vw"] for p in passes for r in p["windows"])
    slot_px = sum(len(p["windows"]) * p["slot"][0] * p["slot"][1] for p in passes)
    res["plan"] = {"windows": sum(len(p["windows"]) for p in passes), "passes": len(passes),
                   "slot_pixels_over_window_pixels": round(slot_px / win_px, 3)}
    if "untiled" not in arms:
        res["untiled"] = f"skipped: its activations alone need {untiled_bytes / 1e9:.0f} GB"

    # bits: outputs and input gradients of the two windowed arms
    got = {}
    for k in ("ragged_tiled", "per_item"):
        outs = arms[k]()
        torch.cuda.synchronize()
        got[k] = [o.detach().clone() for o in outs], [t.grad.clone() for t in leaves]
    a, b = got["ragged_tiled"], got["per_item"]
    res["bitwise_equal_outputs_and_input_grads"] = (all(torch.equal(x, y) for x, y in zip(a[0], b[0])) and
                                                    all(torch.equal(x, y) for x, y in zip(a[1], b[1])))
    del got, a, b

    for _ in range(args.warmup):
        for fn in arms.values():
            fn()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            times[k].append(timed_step_ms(fn))
    for k, fn in arms.items():
        torch.cuda.empty_cache()
        before = eng.launch_count
        fn()
        torch.cuda.synchronize()
        launches = eng.launch_count - before
        med = statistics.median(times[k])
        res[k] = {"ms_per_step": round(med, 2), "ms": [round(t, 2) for t in times[k]],
                  "mpx_per_s": round(total_px / 1e6 / (med / 1e3), 2), "peak_bytes": peak_step_bytes(fn),
                  "launches": launches}
    res["ragged_tiled_vs_per_item"] = round(res["ragged_tiled"]["ms_per_step"] / res["per_item"]["ms_per_step"], 3)
    model.grad_tile = None
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--tile", type=int, default=998)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged_tiled_train.py needs a CUDA device (H100)")
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet().cuda().train()
    res = {"metric": "ragged_windowed_training_step", **card(), "rounds": args.rounds, "grad_tile": args.tile,
           "step": "forward + mse + backward (34 parameter and all input gradients), no VGG"}
    for name, sizes in workloads(args.seed).items():
        res[name] = run(model, sizes, args)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
