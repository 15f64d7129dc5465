"""The native VGG19 perceptual loss in its two arithmetics, bf16x3 (the default) against single-pass bf16
(PerceptualModel.precision), beside the torch expression; prints one JSON line.

    python tools/bench_perceptual_precision.py [--rounds 5] [--warmup 2] [--seed 0]

Workloads:
  loss_4x1080p   loss + d(out) of 4 x 1080p, with one window per image and at tile 998: the torch expression (cuDNN,
                 TF32 as torch defaults it), native bf16x3 and native bf16, arms alternated over --rounds after --warmup
                 calls each.  Per arm: median ms, peak device memory of one call, the VGG convolutions' kernel ms (the
                 handle's timing slot 22, wn_enable_timing) and their share of the call, and the relative differences
                 of the loss and of d(out) (||G - T|| / ||T||) to the torch arm.
  step_*         the full training step of WaterNet(train_precision="bf16"): forward, 0.05 * perc + mse, backward (no
                 optimizer), with the native loss in bf16x3 against bf16, alternated: 16 x 112 x 112 untiled, and
                 4 x 1080p at grad_tile=998 with PerceptualModel(tile=998).  Per arm: median ms, peak memory, the VGG
                 convolutions' kernel ms and their share of the step.
The card's name, power limit and SM clock limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_tiled_train import peak_step_bytes, timed_step_ms  # noqa: E402

VGG_SLOT = 22  # kSlotPost: every VGG convolution launch (csrc/vgg.cu)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:  # noqa: BLE001 -- the numbers stay valid, only unlabelled
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e.__class__.__name__})"}


def vgg_slot_ms(vgg, x, fn):
    """ms of the VGG convolution launches in one call of fn (the VGG engine's timing slot)."""
    eng = vgg._vgg_engine(x)
    eng.enable_timing(True)
    eng.read_timings()
    fn()
    torch.cuda.synchronize()
    ms, cnt = eng.read_timings()
    eng.enable_timing(False)
    return ms[VGG_SLOT] if cnt[VGG_SLOT] else 0.0


def alternated(fns, args):
    for fn in fns.values():
        for _ in range(args.warmup):
            fn()
    ms = {k: [] for k in fns}
    for _ in range(args.rounds):
        for k, fn in fns.items():
            ms[k].append(timed_step_ms(fn))
    return ms


def loss_workload(args, T):
    n, h, w = 4, 1080, 1920
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    out = torch.rand((n, 3, h, w), device="cuda", generator=g)
    ref = (out + 0.2 * torch.rand((n, 3, h, w), device="cuda", generator=g)).clamp(0, 1)
    torch.manual_seed(1234)
    vgg_t = T.PerceptualModel(pretrained=False).cuda().eval()
    arms = {"torch": vgg_t}
    for tile in (None, 998):
        for precision in ("bf16x3", "bf16"):
            v = T.PerceptualModel(pretrained=False, native=True, tile=tile, precision=precision).cuda().eval()
            v.load_state_dict(vgg_t.state_dict())
            arms[f"native_{precision}_tile_{tile}"] = v
    grads = {}

    def call(name):
        def fn():
            o = out.clone().requires_grad_(True)
            loss = T.perceptual_loss(arms[name], o, ref)
            loss.backward()
            grads[name] = (loss.detach(), o.grad)
            arms[name].zero_grad(set_to_none=True)
        return fn
    fns = {k: call(k) for k in arms}
    ms = alternated(fns, args)
    res = {}
    lt, gt = grads["torch"]
    for name in arms:
        med = statistics.median(ms[name])
        lo, go = grads[name]
        r = {"ms": round(med, 1), "spread_ms": [round(min(ms[name]), 1), round(max(ms[name]), 1)],
             "peak_gb": round(peak_step_bytes(fns[name]) / 1e9, 2),
             "loss_rel_diff": float(abs(lo - lt) / abs(lt)),
             "grad_rel_diff": float((go.double() - gt.double()).norm() / gt.double().norm())}
        if name != "torch":
            conv = vgg_slot_ms(arms[name], out, fns[name])
            r["vgg_conv_ms"] = round(conv, 1)
            r["vgg_conv_share"] = round(conv / med, 3)
        res[name] = r
    for tile in (None, 998):
        a, b = res[f"native_bf16_tile_{tile}"], res[f"native_bf16x3_tile_{tile}"]
        res[f"bf16_over_bf16x3_tile_{tile}"] = {"ms": round(a["ms"] / b["ms"], 3),
                                                "vgg_conv_ms": round(a["vgg_conv_ms"] / b["vgg_conv_ms"], 3)}
        lb, gb = grads[f"native_bf16_tile_{tile}"]
        lx, gx = grads[f"native_bf16x3_tile_{tile}"]
        res[f"bf16_vs_bf16x3_tile_{tile}"] = {
            "loss_rel_diff": float(abs(lb - lx) / abs(lx)),
            "grad_rel_diff": float((gb.double() - gx.double()).norm() / gx.double().norm())}
    return {"frames": [n, h, w], "arms": res}


def step_workload(args, T, n, h, w, grad_tile):
    from waternet_b200.net import WaterNet
    g = torch.Generator(device="cuda").manual_seed(args.seed)
    ins = [torch.rand((n, 3, h, w), device="cuda", generator=g) for _ in range(4)]
    ref = torch.rand((n, 3, h, w), device="cuda", generator=g)
    torch.manual_seed(0)
    model = WaterNet(train_precision="bf16", grad_tile=grad_tile).cuda().train()
    vggs = {}
    for precision in ("bf16x3", "bf16"):
        torch.manual_seed(1234)
        vggs[precision] = T.PerceptualModel(pretrained=False, native=True, tile=grad_tile,
                                            precision=precision).cuda().eval()

    def step(precision):
        def fn():
            model.zero_grad(set_to_none=True)
            out = model(*ins)
            loss, _, _ = T.batch_losses(vggs[precision], out, ref)
            loss.backward()
        return fn
    fns = {p: step(p) for p in vggs}
    ms = alternated(fns, args)
    res = {}
    for p in vggs:
        med = statistics.median(ms[p])
        conv = vgg_slot_ms(vggs[p], ref, fns[p])
        res[p] = {"ms": round(med, 1), "spread_ms": [round(min(ms[p]), 1), round(max(ms[p]), 1)],
                  "peak_gb": round(peak_step_bytes(fns[p]) / 1e9, 2), "vgg_conv_ms": round(conv, 1),
                  "vgg_conv_share": round(conv / med, 3)}
    res["bf16_over_bf16x3"] = round(res["bf16"]["ms"] / res["bf16x3"]["ms"], 3)
    return {"frames": [n, h, w], "grad_tile": grad_tile, "arms": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_perceptual_precision.py needs a CUDA device (H100)")
    from waternet_b200 import training as T
    res = {"bench": "perceptual_precision", **card(), "rounds": args.rounds,
           "loss_4x1080p": loss_workload(args, T)}
    torch.cuda.empty_cache()
    res["step_16x112x112"] = step_workload(args, T, 16, 112, 112, None)
    torch.cuda.empty_cache()
    res["step_4x1080p_tile998"] = step_workload(args, T, 4, 1080, 1920, 998)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
