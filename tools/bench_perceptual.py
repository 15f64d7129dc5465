"""The VGG19 perceptual loss on the tensor cores in windows (PerceptualModel(native=True)) against the torch expression
train.py builds; prints one JSON line.

    python tools/bench_perceptual.py [--rounds 3] [--warmup 1] [--seed 0]

Workloads:
  loss_4x1080p     loss + d(out) of 4 x 1080p: native with tile None and 998 against perceptual_loss with the torch
                   VGG19 (cuDNN, TF32 as torch defaults it), arms alternated over --rounds after --warmup calls each.
                   Reported: median ms, peak device memory of one call, and the relative differences of the loss and of
                   d(out) (||G - T|| / ||T||) to the torch arm.
  step_*           the full training step WaterNet(grad_tile=998) -> 0.05 * perc + mse -> backward (no optimizer) with
                   the native loss (tile 998) at 16 x 1080p and 1 x 45 MP: ms, Mpx/s, peak memory.  The torch arm is not
                   run there; its size is given as the bytes autograd would save for the perceptual term (1,564 B per
                   input pixel with frozen VGG parameters, 3,120 B as PerceptualModel's trainable ones are).
The card's name and power limit are read in the same run.
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
from bench_tiled_train import peak_step_bytes, timed_step_ms  # noqa: E402

SAVED_BYTES_PER_PIXEL = 3120  # torch expression, trainable VGG parameters (counted with saved_tensors_hooks)


def loss_workload(args, T):
    n, h, w = 4, 1080, 1920
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    out = torch.rand((n, 3, h, w), device="cuda", generator=g)
    ref = (out + 0.2 * torch.rand((n, 3, h, w), device="cuda", generator=g)).clamp(0, 1)
    torch.manual_seed(1234)
    vgg_t = T.PerceptualModel(pretrained=False).cuda().eval()
    arms = {"torch": vgg_t}
    for tile in (None, 998):
        v = T.PerceptualModel(pretrained=False, native=True, tile=tile).cuda().eval()
        v.load_state_dict(vgg_t.state_dict())
        arms["native_tile_" + str(tile)] = v
    grads = {}

    def call(name):
        def fn():
            o = out.clone().requires_grad_(True)
            loss = T.perceptual_loss(arms[name], o, ref)
            loss.backward()
            grads[name] = (loss.detach(), o.grad)
            arms[name].zero_grad(set_to_none=True)
        return fn
    for name in arms:
        for _ in range(args.warmup):
            call(name)()
    ms = {k: [] for k in arms}
    for _ in range(args.rounds):
        for name in arms:
            ms[name].append(timed_step_ms(call(name)))
    res = {}
    lt, gt = grads["torch"]
    for name in arms:
        peak = peak_step_bytes(call(name))
        lo, go = grads[name]
        res[name] = {"ms": round(statistics.median(ms[name]), 1), "peak_gb": round(peak / 1e9, 2),
                     "loss_rel_diff": float(abs(lo - lt) / abs(lt)),
                     "grad_rel_diff": float((go.double() - gt.double()).norm() / gt.double().norm())}
    return {"frames": [n, h, w], "arms": res}


def step_workload(args, T, n, h, w):
    from waternet_b200.net import WaterNet
    model = WaterNet().cuda().train()
    model.grad_tile = 998
    vgg = T.PerceptualModel(pretrained=False, native=True, tile=998).cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    ins = [torch.rand((n, 3, h, w), device="cuda", generator=g) for _ in range(4)]
    ref = torch.rand((n, 3, h, w), device="cuda", generator=g)

    def step():
        model.zero_grad(set_to_none=True)
        out = model(*ins)
        loss, _, _ = T.batch_losses(vgg, out, ref)
        loss.backward()
    for _ in range(args.warmup):
        step()
    ms = [timed_step_ms(step) for _ in range(args.rounds)]
    med = statistics.median(ms)
    return {"frames": [n, h, w], "ms": round(med, 1), "mpx_s": round(n * h * w / 1e6 / (med / 1e3), 2),
            "peak_gb": round(peak_step_bytes(step) / 1e9, 2),
            "torch_perceptual_saved_gb_derived": round(n * h * w * SAVED_BYTES_PER_PIXEL / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_perceptual.py needs a CUDA device (H100)")
    from waternet_b200 import training as T
    res = {"bench": "perceptual", **card(), "loss_4x1080p": loss_workload(args, T)}
    torch.cuda.empty_cache()
    res["step_16x1080p"] = step_workload(args, T, 16, 1080, 1920)
    torch.cuda.empty_cache()
    res["step_45mp"] = step_workload(args, T, 1, 5792, 7760)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
