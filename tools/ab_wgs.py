#!/usr/bin/env python
"""A/B of two or more builds of the library in one process tree, on the flagship benchmark.

    python -m waternet_b200.build                                            # the product library
    python -c "import waternet_b200.build as b; b.build(defines=('WN_UMMA_WGS2',), lib_name='libwaternet_b200_wgs2.so')"
    python tools/ab_wgs.py --rounds 3 --out <dir>                            # wgs2 against product, identical outputs
    python tools/ab_wgs.py --arm parent=<lib> --arm product=<lib> --u8-tolerance 1 --rounds 3 --out <dir>

Runs `bench.py --gpus 1 --steps 30 --warmup 5 --dump-outputs ...` on each arm in turn (the first arm is the baseline),
`--rounds` times, then once per `--extra` library.  Every run's dumped uint8 images must be within `--u8-tolerance`
of the first run's (0: byte-identical); the largest difference and the fraction of differing bytes are reported.
Without `--arm` the arms are the WN_UMMA_WGS2 library and the product library.  Prints one JSON line with the card
name, power limit and maximum SM clock, and each run's value, clocks, gpu_launches, parity and kernel_ms_per_step;
the same line is written to <out>/ab_wgs.json.
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "waternet_b200")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              "0"], capture_output=True, text=True, check=True).stdout.strip()
        name, power, clock = [f.strip() for f in out.split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except (OSError, subprocess.CalledProcessError, ValueError) as e:
        return {"error": str(e)[:200]}


def run(lib, dump_dir, steps, warmup):
    env = dict(os.environ, WATERNET_B200_LIB=lib)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--dump-outputs", dump_dir]
    res = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [l for l in res.stdout.splitlines() if l.startswith("{")]
    if res.returncode != 0 or not lines:
        raise SystemExit(f"bench.py failed on {lib} (exit {res.returncode}):\n{res.stdout[-2000:]}\n{res.stderr[-4000:]}")
    return json.loads(lines[-1])


def read_dump(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


def dump_diff(a, b):
    """(largest difference, fraction of differing values) of the uint8 images two dumps hold (bench.py stores them as
    float32 .npy files); None when their files or shapes differ."""
    if a.keys() != b.keys():
        return None
    x = [np.load(io.BytesIO(a[f])) for f in a]
    y = [np.load(io.BytesIO(b[f])) for f in b]
    if any(u.shape != v.shape for u, v in zip(x, y)):
        return None
    d = np.concatenate([np.abs(u.astype(np.float64) - v).reshape(-1) for u, v in zip(x, y)])
    return float(d.max(initial=0)), float((d != 0).mean()) if d.size else 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", required=True)
    ap.add_argument("--arm", action="append", default=[], metavar="NAME=LIB",
                    help="an arm of the alternation (the first is the baseline); default: wgs2 and product")
    ap.add_argument("--u8-tolerance", type=int, default=0, help="largest allowed uint8 output difference to run 1")
    ap.add_argument("--extra", action="append", default=[], metavar="NAME=LIB",
                    help="one more run on another build of the library, e.g. one made from an earlier commit")
    args = ap.parse_args()
    arms = {"wgs2": os.path.join(PKG, "libwaternet_b200_wgs2.so"), "product": os.path.join(PKG, "libwaternet_b200.so")}
    if args.arm:
        arms = {name: os.path.abspath(lib) for name, lib in (spec.split("=", 1) for spec in args.arm)}
    for name, lib in arms.items():
        if not os.path.exists(lib):
            raise SystemExit(f"{lib} is missing ({name}); build it first (see the docstring)")
    os.makedirs(args.out, exist_ok=True)
    info = {"card": card(), "steps": args.steps, "warmup": args.warmup, "u8_tolerance": args.u8_tolerance, "runs": []}
    base, new = list(arms)[0], list(arms)[-1]
    order = [(name, r) for r in range(args.rounds) for name in arms]
    for spec in args.extra:
        name, lib = spec.split("=", 1)
        arms[name] = os.path.abspath(lib)
        order.append((name, 0))
    first = None
    for name, r in order:
        dump = os.path.join(args.out, f"{name}_{r}")
        line = run(arms[name], dump, args.steps, args.warmup)
        got = read_dump(dump)
        first = got if first is None else first
        diff = dump_diff(first, got)
        clocks = line.get("clocks") or {}
        info["runs"].append({"arm": name, "round": r, "value": line["value"], "ms_per_step": line["ms_per_step"],
                             "clocks": {k: clocks.get(k) for k in ("sm_mhz", "sm_max_mhz", "power_w_max", "reasons")},
                             "gpu_launches": line["gpu_launches"], "parity": line["parity"],
                             "kernel_ms_per_step": line["kernel_ms_per_step"],
                             "u8_diff_to_first_run": diff,
                             "outputs_within_tolerance": diff is not None and diff[0] <= args.u8_tolerance})
        print(f"{name} {r}: {line['value']:.2f} images/s", file=sys.stderr, flush=True)
    vals = {a: [x["value"] for x in info["runs"] if x["arm"] == a] for a in arms}
    info["summary"] = {
        "images_per_s": vals,
        "baseline": base, "new": new,
        "median_gain": statistics.median(vals[new]) / statistics.median(vals[base]) - 1.0,
        "slowest_new_beats_fastest_baseline": min(vals[new]) > max(vals[base]),
        "all_outputs_within_tolerance": all(x["outputs_within_tolerance"] for x in info["runs"]),
        "gpu_launches": sorted({x["gpu_launches"] for x in info["runs"]}),
        # per arm, the slots its runs timed (a launch one build fuses away has no slot there)
        "kernel_ms_per_step_median": {a: {k: statistics.median(x["kernel_ms_per_step"][k] for x in info["runs"]
                                                               if x["arm"] == a and k in x["kernel_ms_per_step"])
                                          for k in dict.fromkeys(k for x in info["runs"] if x["arm"] == a
                                                                 for k in x["kernel_ms_per_step"])} for a in arms},
    }
    line = json.dumps(info)
    with open(os.path.join(args.out, "ab_wgs.json"), "w") as f:
        f.write(line + "\n")
    print(line, flush=True)
    if not info["summary"]["all_outputs_within_tolerance"]:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
