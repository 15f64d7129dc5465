"""SSIM + PSNR of a batch, the torch expression (``training.batch_quality``) against the native path
(``batch_quality(native=True)``, one ``wn_quality`` call), on one GPU; prints one JSON line.

    python tools/bench_metrics.py [--rounds 5] [--calls 10]

Cases: 16 x 112 x 112 (train.py's default batch), 16 x 1080p, a ragged list of 32 mixed sizes (64..1080 per side),
and 1 x 8256 x 5504 (a 45 MP photo).  Per case: ms per call of each path (CUDA events around --calls calls, after a
warm-up, over --rounds alternated rounds; the median), the peak device memory each call adds above its inputs, and
native's time against the lower bound of its SSIM launch: 24 B per pixel read from HBM (out and ref, 3 fp32 planes)
at 3.35 TB/s, or ~660 fp32 flop per pixel (22 taps x 5 moments x 3 planes x 2) at 67 TFLOP/s, whichever is larger --
the H100 SXM data sheet, not a target.  Then the train.py-style windowed step at 4 x 1080p (``grad_tile=998``, the
native VGG loss in windows of 998, ``0.05 * perc + mse``, backward, Adam) with each metric path after it: ms per
step and peak memory.  The card's name and power limit are read in the same run; they belong beside every number.
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

HBM_BYTES_PER_S = 3.35e12
FP32_FLOP_PER_S = 67e12
BYTES_PER_PX, FLOP_PER_PX = 24, 660


def _pair(n, h, w, g):
    a = torch.rand((n, 3, h, w), generator=g, device="cuda")
    return a, (a + 0.05 * torch.randn((n, 3, h, w), generator=g, device="cuda")).clamp_(0, 1)


def cases():
    g = torch.Generator(device="cuda").manual_seed(0)
    sizes = [(64 + (k * 97) % 1017, 64 + (k * 211) % 1017) for k in range(32)]
    ragged = [_pair(1, h, w, g) for h, w in sizes]
    return {
        "16x112x112": _pair(16, 112, 112, g),
        "16x1080p": _pair(16, 1080, 1920, g),
        "ragged32": ([o for o, _ in ragged], [r for _, r in ragged]),
        "1x45MP": _pair(1, 5504, 8256, g),
    }


def pixels(out):
    return sum(o[:, 0].numel() for o in out) if isinstance(out, list) else out[:, 0].numel()


def timed_ms(fn, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def peak_added(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def bench_case(out, ref, rounds, calls):
    from waternet_b200 import training as T
    paths = {"torch": lambda: T.batch_quality(out, ref), "native": lambda: T.batch_quality(out, ref, native=True)}
    res = {}
    for name, fn in paths.items():
        fn()  # warm-up
        res[name] = {"peak_added_mb": round(peak_added(fn) / 2 ** 20, 1), "ms": []}
    for _ in range(rounds):
        for name, fn in paths.items():
            res[name]["ms"].append(timed_ms(fn, calls))
    for name in paths:
        res[name]["ms"] = round(statistics.median(res[name]["ms"]), 3)
    px = pixels(out)
    bound_ms = max(px * BYTES_PER_PX / HBM_BYTES_PER_S, px * FLOP_PER_PX / FP32_FLOP_PER_S) * 1e3
    s_t, p_t = (v.item() for v in paths["torch"]())
    s_n, p_n = (v.item() for v in paths["native"]())
    res.update(pixels=px, native_over_torch=round(res["native"]["ms"] / res["torch"]["ms"], 3),
               ssim_bound_ms=round(bound_ms, 3),
               ssim_bound_by="hbm" if BYTES_PER_PX / HBM_BYTES_PER_S > FLOP_PER_PX / FP32_FLOP_PER_S else "fp32",
               bound_over_native=round(bound_ms / res["native"]["ms"], 3),
               ssim_diff=abs(s_t - s_n), psnr_diff=abs(p_t - p_n))
    return res


def bench_step(rounds):
    """The windowed step of train.py at 4 x 1080p followed by each metric path."""
    from waternet.net import WaterNet
    from waternet_b200 import training as T
    torch.manual_seed(0)
    model = WaterNet().cuda().train()
    model.grad_tile = 998
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    vgg = T.PerceptualModel(pretrained=False, native=True, tile=998).cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    ins = [torch.rand((4, 3, 1080, 1920), generator=g, device="cuda") for _ in range(4)]
    ref = torch.rand((4, 3, 1080, 1920), generator=g, device="cuda")

    def step(native):
        out = model(*ins)
        loss, _, _ = T.batch_losses(vgg, out, ref)
        opt.zero_grad()
        loss.backward()
        opt.step()
        with torch.no_grad():
            s, p = T.batch_quality(out, ref, native)
            s.item(), p.item()

    res = {}
    for native in (False, True):
        step(native)
        res["native" if native else "torch"] = {"peak_gb": round(peak_added(lambda: step(native)) / 2 ** 30, 2),
                                                "ms": []}
    for _ in range(rounds):
        for native in (False, True):
            res["native" if native else "torch"]["ms"].append(timed_ms(lambda: step(native), 1))
    for k in res:
        res[k]["ms"] = round(statistics.median(res[k]["ms"]), 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--step-rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_metrics.py needs a CUDA device")
    result = {"bench": "metrics", **card(), "cases": {}}
    for name, (out, ref) in cases().items():
        result["cases"][name] = bench_case(out, ref, args.rounds, args.calls)
        del out, ref
        torch.cuda.empty_cache()
    result["step_4x1080p_grad_tile998"] = bench_step(args.step_rounds)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
