"""Windowed (``grad_tile``) against untiled training steps of one sub-module called on its own; prints one JSON line.

    python tools/bench_submodule_tiled_train.py [--rounds 3] [--warmup 1] [--grad-tile 998]

A step is forward, MSE against a random target, and backward with the gradients of the sub-module's parameters and of
its input images (no optimizer), timed with CUDA events after warm-up.  Sub-modules: ``model.cmg`` and
``model.ce_refiner`` of a default-initialised WaterNet.  At 2 x 1080p both paths run, alternated over --rounds: ms per
step, peak device memory of one step, their step-time ratio and the worst relative difference of the parameter
gradients between them (max |a - b| / max |b| per tensor).  Then the windowed path alone at 16 x 1080p and at
1 x 5504 x 8256 (a 45 MP photo, over the untiled call's limit).  For every windowed case the forward alone is timed
too (``fwd_ms``: the tiled forward that the step's backward does not reuse).  The card's name and power limit are read
in the same run; they belong beside every number.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_tiled import card  # noqa: E402
from bench_tiled_train import peak_step_bytes, row, timed_step_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--grad-tile", type=int, default=998)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_submodule_tiled_train.py needs a CUDA device (H100)")
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet().cuda().train()
    tile = args.grad_tile
    res = {"metric": "submodule_windowed_vs_untiled_training_step", **card(), "grad_tile": tile,
           "rounds": args.rounds, "step": "forward + mse + backward (parameter and input gradients), no optimizer"}

    def data(n, h, w):
        gen = torch.Generator(device="cuda").manual_seed(n * h + w)
        return ([torch.rand(n, 3, h, w, device="cuda", generator=gen).requires_grad_(True) for _ in range(4)],
                torch.rand(n, 3, h, w, device="cuda", generator=gen))

    def fns(name, ins, target):
        mod = getattr(model, name)

        def call():
            return torch.cat(mod(*ins), 1) if name == "cmg" else mod(ins[0], ins[2])

        def step():
            mod.zero_grad(set_to_none=True)
            for t in ins:
                t.grad = None
            F.mse_loss(call(), target).backward()

        return mod, call, step

    def timed_ms(fn):  # every switch of path starts from an empty cache, outside the timed region
        torch.cuda.empty_cache()
        return timed_step_ms(fn)

    def fwd_ms(call):
        return round(statistics.median(timed_step_ms(call) for _ in range(args.rounds)), 1)

    # ---- 2 x 1080p: both paths, alternated
    n, h, w = 2, 1080, 1920
    ins, target = data(n, h, w)
    for name in ("cmg", "ce_refiner"):
        mod, call, step = fns(name, ins, target)

        def untiled(step=step):
            model.grad_tile = None
            step()

        def tiled(step=step):
            model.grad_tile = tile
            step()

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
        g_u = [p.grad.clone() for p in mod.parameters()]
        torch.cuda.empty_cache()
        tiled()
        g_t = [p.grad.clone() for p in mod.parameters()]
        worst = max(((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item() for a, b in zip(g_t, g_u))
        del g_u, g_t
        torch.cuda.empty_cache()
        p_u = peak_step_bytes(untiled)
        torch.cuda.empty_cache()
        p_t = peak_step_bytes(tiled)
        model.grad_tile = tile
        res[f"{name}_2x1080p"] = {"untiled": {**row(n, h, w, t_u), "peak_bytes": p_u},
                                  "grad_tile": {**row(n, h, w, t_t), "peak_bytes": p_t, "fwd_ms": fwd_ms(call)},
                                  "step_ratio": round(statistics.median(t_t) / statistics.median(t_u), 3),
                                  "worst_grad_rel_diff": worst}
        mod.zero_grad(set_to_none=True)
    del ins, target
    torch.cuda.empty_cache()

    # ---- windowed alone where the untiled call does not fit or is refused
    model.grad_tile = tile
    lib = model.engine().lib
    for key, (n, h, w) in (("16x1080p", (16, 1080, 1920)), ("45mp", (1, 5504, 8256))):
        ins, target = data(n, h, w)
        for name, stack in (("cmg", 0), ("ce_refiner", 1)):
            mod, call, step = fns(name, ins, target)
            for _ in range(args.warmup):
                step()
            t = [timed_step_ms(step) for _ in range(args.rounds)]
            res[f"{name}_{key}"] = {**row(n, h, w, t), "peak_bytes": peak_step_bytes(step), "fwd_ms": fwd_ms(call),
                                    "untiled_activation_bytes": n * h * w * (3852 if stack == 0 else 1828)}
            mod.zero_grad(set_to_none=True)
        del ins, target
        torch.cuda.empty_cache()
    res["workspace_bytes_default_pass"] = {
        "cmg": int(lib.wn_submodule_backward_tiled_workspace_bytes(1, 5504, 8256, tile, tile, 0, 0)),
        "refiner": int(lib.wn_submodule_backward_tiled_workspace_bytes(1, 5504, 8256, tile, tile, 0, 1))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
