"""Windowed (``WaterNet.grad_tile``) against untiled training steps on one GPU; prints one JSON line.

    python tools/bench_tiled_train.py [--rounds 3] [--warmup 1] [--grad-tile 998]

A step is forward + backward of the 34 WaterNet parameters with an MSE loss against a random target, no VGG and no
optimizer (as tools/bench_train.py), timed with CUDA events after warm-up.  4 x 1080p runs both ways, alternated
over --rounds: ms per step, Mpx/s, peak device memory of each, their step-time ratio and the worst relative
difference of the 34 gradients between the two paths (max |a - b| / max |b| per tensor).  Then the windowed path
alone at 16 x 1080p (bench.py's batch, 186 GB of activations untiled) and at 1 x 8256x5504 (a 45 MP photo, which the
untiled path refuses).  The card's name and power limit are read in the same run; they belong beside every number.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_tiled import card  # noqa: E402


def step_fn(model, ins, target):
    def step():
        model.zero_grad(set_to_none=True)
        torch.nn.functional.mse_loss(model(*ins), target).backward()
    return step


def timed_step_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak_step_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return int(torch.cuda.max_memory_allocated())


def row(n, h, w, ms):
    return {"frames": [n, h, w], "ms_per_step": round(statistics.median(ms), 1), "ms": [round(t, 1) for t in ms],
            "mpx_s": round(n * h * w / 1e6 / (statistics.median(ms) / 1e3), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--grad-tile", type=int, default=998)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiled_train.py needs a CUDA device (H100)")
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet().cuda().train()  # default init; training runs the bf16x3 arithmetic
    tile = args.grad_tile
    res = {"metric": "windowed_vs_untiled_training_step", **card(), "grad_tile": tile, "rounds": args.rounds,
           "loss": "mse, no vgg, no optimizer"}

    def data(n, h, w):
        gen = torch.Generator(device="cuda").manual_seed(n * h + w)
        return ([torch.rand(n, 3, h, w, device="cuda", generator=gen) for _ in range(4)],
                torch.rand(n, 3, h, w, device="cuda", generator=gen))

    # ---- 4 x 1080p: both paths, alternated
    n, h, w = 4, 1080, 1920
    ins, target = data(n, h, w)
    step = step_fn(model, ins, target)

    # the untiled step allocates one 43 GB workspace per call; the windowed step's smaller blocks would split the
    # cached one, so every switch of path starts from an empty cache (outside the timed region)
    def untiled():
        model.grad_tile = None
        step()

    def tiled():
        model.grad_tile = tile
        step()

    def timed_ms(fn):
        torch.cuda.empty_cache()
        return timed_step_ms(fn)

    def peak_bytes(fn):
        torch.cuda.empty_cache()
        return peak_step_bytes(fn)

    for _ in range(args.warmup):
        for fn in (untiled, tiled):
            torch.cuda.empty_cache()
            fn()
    t_u, t_t = [], []
    for _ in range(args.rounds):
        t_u.append(timed_ms(untiled))
        t_t.append(timed_ms(tiled))
    torch.cuda.empty_cache()
    untiled()
    g_u = [p.grad.clone() for p in model.parameters()]
    torch.cuda.empty_cache()
    tiled()
    g_t = [p.grad.clone() for p in model.parameters()]
    worst = max(((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item() for a, b in zip(g_t, g_u))
    del g_u, g_t
    p_u, p_t = peak_bytes(untiled), peak_bytes(tiled)
    res["4x1080p"] = {"untiled": {**row(n, h, w, t_u), "peak_bytes": p_u},
                      "grad_tile": {**row(n, h, w, t_t), "peak_bytes": p_t},
                      "step_ratio": round(statistics.median(t_t) / statistics.median(t_u), 3),
                      "worst_grad_rel_diff": worst}
    del ins, target, step
    model.zero_grad(set_to_none=True)
    torch.cuda.empty_cache()

    # ---- windowed alone where the untiled path does not fit
    model.grad_tile = tile
    for key, (n, h, w) in (("16x1080p", (16, 1080, 1920)), ("45mp", (1, 5504, 8256))):
        ins, target = data(n, h, w)
        step = step_fn(model, ins, target)
        for _ in range(args.warmup):
            step()
        t = [timed_step_ms(step) for _ in range(args.rounds)]
        res[key] = {**row(n, h, w, t), "peak_bytes": peak_step_bytes(step),
                    "untiled_activation_bytes": int(model.engine().lib.wn_train_workspace_bytes(n, h, w))}
        del ins, target, step
        model.zero_grad(set_to_none=True)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
