"""Tiled vs whole-image enhance on one GPU; prints one JSON line.

    python tools/bench_tiled.py [--rounds 3] [--warmup 2] [--mode default]

4 x 3840x2160 frames through Engine.enhance (whole images per pass) and Engine.enhance_tiled (998 x 998 tiles),
timed with CUDA events, alternated over --rounds, both warmed up first: Mpx/s of each, their ratio, the geometric
recompute factor of the windows, each path's workspace and whether the two outputs are bitwise equal.  Then
2 x 7680x4320 frames on the tiled path only (untiled they would need 62 GB of workspace).  Per-kernel times of one
call of each path (wn_enable_timing) are included to explain the ratio.  The card's name and power limit are read
with an nvidia-smi query; they belong beside every number this prints.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLOTS = {17: "pack", 18: "gate", 19: "stats", 20: "luts", 21: "apply", 22: "post"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers stay valid, only unlabelled
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e.__class__.__name__})"}


def frames(n, h, w, seed):
    """Blue-green underwater-like frames: low-frequency structure + noise (deterministic), built on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    coarse = torch.rand((n, 3, h // 40 + 2, w // 40 + 2), generator=g, device="cuda")
    up = torch.nn.functional.interpolate(coarse, scale_factor=40, mode="nearest")[:, :, :h, :w]
    img = up * torch.tensor([90.0, 200.0, 230.0], device="cuda")[None, :, None, None]
    img = img + torch.randint(0, 24, (n, 3, h, w), generator=g, device="cuda")
    return img.clamp(1, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def kernel_ms(eng, fn):
    eng.enable_timing(True)
    fn()
    ms, cnt = eng.read_timings()
    eng.enable_timing(False)
    convs = sum(ms[:17])
    return {"conv": round(convs, 2), **{name: round(ms[s], 2) for s, name in SLOTS.items() if cnt[s]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--mode", choices=["default", "bf16x3", "bf16_fp8"], default="default")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiled.py needs a CUDA device (H100)")
    from waternet_b200.engine import tile_geometry
    from waternet_b200.net import WaterNet

    torch.manual_seed(0)
    model = WaterNet(precision=args.mode).cuda().eval()  # default init, as bench.py
    eng = model.engine()
    mode = model._mode()
    tile = eng.DEFAULT_TILE
    res = {"metric": "tiled_vs_untiled_enhance", **card(), "mode": args.mode, "tile": list(tile),
           "rounds": args.rounds}

    n, h, w = 4, 2160, 3840
    x = frames(n, h, w, 0)
    u8_a, u8_b = torch.empty_like(x), torch.empty_like(x)
    f32_a, f32_b = [torch.empty(n, 3, h, w, device="cuda") for _ in range(2)]
    untiled = lambda: eng.enhance(x, mode=mode, out_u8=u8_a)
    tiled = lambda: eng.enhance_tiled(x, tile=tile, mode=mode, out_u8=u8_b)
    for _ in range(args.warmup):
        untiled()
        tiled()
    t_a, t_b = [], []
    for _ in range(args.rounds):
        t_a.append(timed(untiled))
        t_b.append(timed(tiled))
    eng.enhance(x, mode=mode, out_u8=u8_a, out_f32=f32_a)
    eng.enhance_tiled(x, tile=tile, mode=mode, out_u8=u8_b, out_f32=f32_b)
    torch.cuda.synchronize()
    g = tile_geometry(h, w, *tile)
    mpx = n * h * w / 1e6
    ra, rb = mpx / statistics.median(t_a), mpx / statistics.median(t_b)
    res["4k"] = {
        "frames": [n, h, w], "untiled_mpx_s": round(ra, 1), "tiled_mpx_s": round(rb, 1), "ratio": round(rb / ra, 3),
        "untiled_s": [round(t, 4) for t in t_a], "tiled_s": [round(t, 4) for t in t_b],
        "recompute_factor": round(len(g["windows"]) * g["win_h"] * g["win_w"] / (h * w), 4),
        "untiled_workspace_bytes": int(eng.lib.wn_enhance_workspace_bytes(n, h, w, mode)),
        "tiled_workspace_bytes": eng.tiled_workspace_bytes(n, h, w, tile, mode),
        "bitwise_equal": bool(torch.equal(u8_a, u8_b) and torch.equal(f32_a, f32_b)),
        "kernel_ms_untiled": kernel_ms(eng, untiled), "kernel_ms_tiled": kernel_ms(eng, tiled),
    }
    del x, u8_a, u8_b, f32_a, f32_b
    eng.release_workspaces()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()

    n, h, w = 2, 4320, 7680
    x = frames(n, h, w, 1)
    out = torch.empty_like(x)
    run = lambda: eng.enhance_tiled(x, tile=tile, mode=mode, out_u8=out)
    for _ in range(args.warmup):
        run()
    t = [timed(run) for _ in range(args.rounds)]
    res["8k"] = {"frames": [n, h, w], "tiled_mpx_s": round(n * h * w / 1e6 / statistics.median(t), 1),
                 "tiled_s": [round(v, 4) for v in t],
                 "tiled_workspace_bytes": eng.tiled_workspace_bytes(n, h, w, tile, mode),
                 "untiled_workspace_bytes": int(eng.lib.wn_enhance_workspace_bytes(n, h, w, mode)),
                 "peak_allocated_bytes": int(torch.cuda.max_memory_allocated())}
    res["f8_overflowed"] = eng.f8_overflowed()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
