"""1 - SSIM and its backward: torch autograd of ``metrics.ssim`` (``batch_quality`` for lists) against
``metrics.ssim_loss`` (one ``wn_ssim_grad`` call), on one GPU; prints one JSON line.

    python tools/bench_ssim_loss.py [--rounds 5] [--calls 5] [--step-rounds 3]

Cases: 16 x 112 x 112 (train.py's default batch), 4 x 1080p, 16 x 1080p, a ragged list of 32 mixed sizes (64..1080
per side) and 1 x 8256 x 5504 (a 45 MP photo).  Per case and path: ms per loss + backward (CUDA events around
--calls calls after a warm-up, the median over --rounds alternated rounds) and the peak device memory the call adds
above its inputs, d(out) included; a path that runs out of memory is recorded as "oom".  Then the train.py-style
windowed step at 4 x 1080p (``grad_tile=998``, the native VGG loss in windows of 998, ``0.05 * perc + mse``,
backward, Adam) without and with ``+ 0.5 * ssim_loss``: ms per step and peak memory.  The card's name and power
limit are read in the same run; they belong beside every number.
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


def _pair(n, h, w, g):
    a = torch.rand((n, 3, h, w), generator=g, device="cuda")
    return a, (a + 0.05 * torch.randn((n, 3, h, w), generator=g, device="cuda")).clamp_(0, 1)


def cases():
    g = torch.Generator(device="cuda").manual_seed(0)
    sizes = [(64 + (k * 97) % 1017, 64 + (k * 211) % 1017) for k in range(32)]
    ragged = [_pair(1, h, w, g) for h, w in sizes]
    yield "16x112x112", _pair(16, 112, 112, g)
    yield "4x1080p", _pair(4, 1080, 1920, g)
    yield "16x1080p", _pair(16, 1080, 1920, g)
    yield "ragged32", ([o for o, _ in ragged], [r for _, r in ragged])
    yield "1x45MP", _pair(1, 5504, 8256, g)


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


def loss_paths(out, ref):
    from waternet_b200 import metrics
    from waternet_b200 import training as T
    leaves = [o.detach().requires_grad_() for o in out] if isinstance(out, list) else out.detach().requires_grad_()

    def run(native):
        if isinstance(leaves, list):
            for t in leaves:
                t.grad = None
            loss = metrics.ssim_loss(leaves, ref) if native else 1 - T.batch_quality(leaves, ref)[0]
        else:
            leaves.grad = None
            loss = metrics.ssim_loss(leaves, ref) if native else 1 - metrics.ssim(leaves, ref)
        loss.backward()
        return loss.item()
    return {"torch": lambda: run(False), "native": lambda: run(True)}


def bench_case(out, ref, rounds, calls):
    paths = loss_paths(out, ref)
    res, ok = {}, {}
    for name, fn in paths.items():
        try:
            fn()  # warm-up
            res[name] = {"peak_added_mb": round(peak_added(fn) / 2 ** 20, 1), "ms": []}
            ok[name] = True
        except torch.OutOfMemoryError:
            res[name] = "oom"
            ok[name] = False
        torch.cuda.empty_cache()
    for _ in range(rounds):
        for name, fn in paths.items():
            if ok[name]:
                res[name]["ms"].append(timed_ms(fn, calls))
    for name in paths:
        if ok[name]:
            res[name]["ms"] = round(statistics.median(res[name]["ms"]), 3)
    res["pixels"] = pixels(out)
    if ok["torch"] and ok["native"]:
        res["native_over_torch"] = round(res["native"]["ms"] / res["torch"]["ms"], 3)
        res["loss_diff"] = abs(paths["torch"]() - paths["native"]())
    return res


def bench_step(rounds):
    """The windowed step of train.py at 4 x 1080p without and with 0.5 * ssim_loss."""
    from waternet.net import WaterNet
    from waternet_b200 import metrics
    from waternet_b200 import training as T
    torch.manual_seed(0)
    model = WaterNet().cuda().train()
    model.grad_tile = 998
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    vgg = T.PerceptualModel(pretrained=False, native=True, tile=998).cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    ins = [torch.rand((4, 3, 1080, 1920), generator=g, device="cuda") for _ in range(4)]
    ref = torch.rand((4, 3, 1080, 1920), generator=g, device="cuda")

    def step(weight):
        out = model(*ins)
        loss, _, _ = T.batch_losses(vgg, out, ref)
        if weight:
            loss = loss + weight * metrics.ssim_loss(out, ref)
        opt.zero_grad()
        loss.backward()
        opt.step()
        loss.item()

    res = {}
    for w in (0.0, 0.5):
        step(w)
        res[f"ssim_weight_{w}"] = {"peak_gb": round(peak_added(lambda: step(w)) / 2 ** 30, 2), "ms": []}
    for _ in range(rounds):
        for w in (0.0, 0.5):
            res[f"ssim_weight_{w}"]["ms"].append(timed_ms(lambda: step(w), 1))
    for k in res:
        res[k]["ms"] = round(statistics.median(res[k]["ms"]), 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--step-rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ssim_loss.py needs a CUDA device")
    result = {"bench": "ssim_loss", **card(), "cases": {}}
    for name, (out, ref) in cases():
        result["cases"][name] = bench_case(out, ref, args.rounds, args.calls)
        del out, ref
        torch.cuda.empty_cache()
    result["step_4x1080p_grad_tile998"] = bench_step(args.step_rounds)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
