"""Training steps of one sub-module called on its own: the native path against the torch graph; prints one JSON line.

    python tools/bench_submodule_train.py [--rounds 5] [--warmup 2]

A step is forward, MSE against a random target, and backward with the gradients of the sub-module's parameters and
of its input images (no optimizer), timed with CUDA events after warm-up.  Sub-modules: ``model.cmg`` and
``model.ce_refiner`` of a default-initialised WaterNet.  Paths, alternated over --rounds: native
(wn_confidence_maps_train / wn_refine_train and their backward), and the torch graph (``_graph()`` over cuDNN) with
TF32 on (torch's default) and off.  Shapes: 16 x 112 x 112 (train.py's batch) and 2 x 1080p.  Reported per case:
median ms per step and peak device memory of one step.  The card's name and power limit are read in the same run;
they belong beside every number.
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
from bench_tiled_train import peak_step_bytes, timed_step_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_submodule_train.py needs a CUDA device (H100)")
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet().cuda().train()
    res = {"metric": "submodule_training_step", **card(), "rounds": args.rounds,
           "step": "forward + mse + backward (parameter and input gradients), no optimizer"}
    tf32 = torch.backends.cudnn.allow_tf32

    for n, h, w in ((16, 112, 112), (2, 1080, 1920)):
        gen = torch.Generator(device="cuda").manual_seed(n * h + w)
        ins = [torch.rand(n, 3, h, w, device="cuda", generator=gen).requires_grad_(True) for _ in range(4)]
        target = torch.rand(n, 3, h, w, device="cuda", generator=gen)
        for name in ("cmg", "ce_refiner"):
            mod = getattr(model, name)

            def call(native, mod=mod, name=name):
                if name == "cmg":
                    return torch.cat(mod(*ins), 1) if native else mod._graph(*ins)
                return mod(ins[0], ins[2]) if native else mod._graph(ins[0], ins[2])

            def step(native, allow_tf32=True, call=call, mod=mod):
                torch.backends.cudnn.allow_tf32 = allow_tf32
                mod.zero_grad(set_to_none=True)
                for t in ins:
                    t.grad = None
                F.mse_loss(call(native), target).backward()

            paths = {"native": lambda: step(True), "graph_tf32": lambda: step(False, True),
                     "graph_fp32": lambda: step(False, False)}
            for _ in range(args.warmup):
                for fn in paths.values():
                    fn()
            times = {k: [] for k in paths}
            for _ in range(args.rounds):
                for k, fn in paths.items():
                    times[k].append(timed_step_ms(fn))
            case = {}
            for k, fn in paths.items():
                torch.cuda.empty_cache()
                case[k] = {"ms_per_step": round(statistics.median(times[k]), 2), "ms": [round(t, 2) for t in times[k]],
                           "peak_bytes": peak_step_bytes(fn)}
            case["native_vs_graph_tf32"] = round(case["native"]["ms_per_step"] / case["graph_tf32"]["ms_per_step"], 3)
            res[f"{name}_{n}x{h}x{w}"] = case
        del ins, target
        torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = tf32
    print(json.dumps(res))


if __name__ == "__main__":
    main()
