"""Tiled vs whole-image forward of fp32 tensors on one GPU; prints one JSON line.

    python tools/bench_tiled_forward.py [--rounds 3] [--warmup 2] [--mode default]

The inputs are the four fp32 tensors of one photo, resident on the device (what the hub model receives).  1 x
3840x2160 through Engine.forward (whole image per pass) and Engine.forward_tiled (998 x 998 tiles), timed with CUDA
events, alternated over --rounds, both warmed up first: Mpx/s of each, their ratio, each path's workspace and
whether the two outputs are bitwise equal.  Then 1 x 8256x5504 (a 45 MP photo) on the tiled path only: untiled it
would need 85 GB of workspace.  Per-kernel times of one call of each (wn_enable_timing) explain the ratio.  The
card's name and power limit are read with an nvidia-smi query; they belong beside every number this prints.
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

from bench_tiled import card, frames, kernel_ms, timed  # noqa: E402


def inputs(eng, n, h, w, seed):
    pre = eng.preprocess(frames(n, h, w, seed))
    return [pre[k] for k in ("x", "wb", "he", "gc")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--mode", choices=["default", "bf16x3", "bf16_fp8"], default="default")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiled_forward.py needs a CUDA device (H100)")
    from waternet_b200.engine import tile_geometry
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet(precision=args.mode).cuda().eval()  # default init, as bench.py
    eng = model.engine()
    mode = model._mode()
    tile = eng.DEFAULT_TILE
    res = {"metric": "tiled_vs_untiled_forward", **card(), "mode": args.mode, "tile": list(tile),
           "rounds": args.rounds}

    n, h, w = 1, 2160, 3840
    ins = inputs(eng, n, h, w, 0)
    out_a, out_b = [torch.empty(n, 3, h, w, device="cuda") for _ in range(2)]
    untiled = lambda: eng.forward(*ins, mode=mode, out=out_a)
    tiled = lambda: eng.forward_tiled(*ins, tile=tile, mode=mode, out=out_b)
    for _ in range(args.warmup):
        untiled()
        tiled()
    t_a, t_b = [], []
    for _ in range(args.rounds):
        t_a.append(timed(untiled))
        t_b.append(timed(tiled))
    torch.cuda.synchronize()
    g = tile_geometry(h, w, *tile)
    mpx = n * h * w / 1e6
    ra, rb = mpx / statistics.median(t_a), mpx / statistics.median(t_b)
    res["4k"] = {
        "frames": [n, h, w], "untiled_mpx_s": round(ra, 1), "tiled_mpx_s": round(rb, 1), "ratio": round(rb / ra, 3),
        "untiled_s": [round(t, 4) for t in t_a], "tiled_s": [round(t, 4) for t in t_b],
        "recompute_factor": round(len(g["windows"]) * g["win_h"] * g["win_w"] / (h * w), 4),
        "untiled_workspace_bytes": int(eng.lib.wn_forward_workspace_bytes(n, h, w, mode)),
        "tiled_workspace_bytes": eng.forward_tiled_workspace_bytes(n, h, w, tile, mode),
        "bitwise_equal": bool(torch.equal(out_a, out_b)),
        "kernel_ms_untiled": kernel_ms(eng, untiled), "kernel_ms_tiled": kernel_ms(eng, tiled),
    }
    del ins, out_a, out_b
    eng.release_workspaces()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()

    n, h, w = 1, 5504, 8256
    ins = inputs(eng, n, h, w, 1)
    out = torch.empty(n, 3, h, w, device="cuda")
    run = lambda: eng.forward_tiled(*ins, tile=tile, mode=mode, out=out)
    for _ in range(args.warmup):
        run()
    t = [timed(run) for _ in range(args.rounds)]
    res["45mp"] = {"frames": [n, h, w], "tiled_mpx_s": round(n * h * w / 1e6 / statistics.median(t), 1),
                   "tiled_s": [round(v, 4) for v in t],
                   "tiled_workspace_bytes": eng.forward_tiled_workspace_bytes(n, h, w, tile, mode),
                   "untiled_workspace_bytes": int(eng.lib.wn_forward_workspace_bytes(n, h, w, mode)),
                   "peak_allocated_bytes": int(torch.cuda.max_memory_allocated()),
                   "kernel_ms_tiled": kernel_ms(eng, run)}
    res["f8_overflowed"] = eng.f8_overflowed()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
