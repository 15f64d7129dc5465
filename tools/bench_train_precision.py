"""Training step in the two training arithmetics: bf16x3 (the default) against single-pass bf16 (train_precision).

One step = forward, MSE against a random target, backward of the parameters (no VGG loss, no optimizer).  Cases: the
reference's training shape 16 x 112 x 112, 4 x 1080p untiled and at grad_tile=998 (the forward of a grad_tile call is
wn_forward_tiled in bf16x3 in both arithmetics: only the recomputed forward and the backward change), and model.cmg and
model.ce_refiner alone at 2 x 1080p.  The two arithmetics and the torch graph with TF32 (cuDNN) run in alternated
rounds of CUDA-event-timed steps after warm-up; per case the median over rounds of ms per step, the per-slot kernel
ms of one native step of each (wn_enable_timing; slots 0..16 = the convolutions in state-dict order, 17 packing,
18 the seeds and data-gradient launches), the peak memory of one step and the ratios.  One JSON line, with the
card's name and power limit.

    python tools/bench_train_precision.py [--rounds 5] [--steps 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from waternet_b200.net import WaterNet  # noqa: E402

CASES = [("waternet", 16, 112, 112, None), ("waternet", 4, 1080, 1920, None), ("waternet", 4, 1080, 1920, 998),
         ("cmg", 2, 1080, 1920, None), ("ce_refiner", 2, 1080, 1920, None)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception:  # noqa: BLE001 -- the numbers stay valid without the label
        return torch.cuda.get_device_name(0), "unknown"


def make_step(m, module, ins, tgt, graph):
    def step():
        m.zero_grad(set_to_none=True)
        if module == "waternet":
            out = m._graph(*ins) if graph else m(*ins)
        elif module == "cmg":
            out = m.cmg._graph(*ins) if graph else torch.cat(m.cmg(*ins), 1)
        else:
            out = m.ce_refiner._graph(ins[0], ins[2]) if graph else m.ce_refiner(ins[0], ins[2])
        torch.nn.functional.mse_loss(out, tgt).backward()
    return step


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 30


def slots(m, fn):
    eng = m.engine()
    eng.enable_timing(True)
    eng.read_timings()
    fn()
    ms, cnt = eng.read_timings()
    eng.enable_timing(False)
    return {str(i): round(v, 3) for i, v in enumerate(ms) if cnt[i]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    name, limit = card()
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    res = []
    for module, n, h, w, grad_tile in CASES:
        ins = [torch.rand(n, 3, h, w, device="cuda") for _ in range(4)]
        tgt = torch.rand(n, 3, h, w, device="cuda")
        models = {tp: WaterNet(train_precision=tp, grad_tile=grad_tile).cuda().train() for tp in ("bf16x3", "bf16")}
        sd = models["bf16x3"].state_dict()
        models["bf16"].load_state_dict(sd)
        steps = {tp: make_step(m, module, ins, tgt, False) for tp, m in models.items()}
        steps["tf32"] = make_step(models["bf16x3"], module, ins, tgt, True)
        for fn in steps.values():  # warm-up: module loads, cuDNN algorithm choice, workspaces
            fn()
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in steps}
        for _ in range(args.rounds):  # alternated rounds
            for k, fn in steps.items():
                times[k].append(timed(fn, args.steps))
        med = {k: statistics.median(v) for k, v in times.items()}
        row = {"module": module, "n": n, "h": h, "w": w, "grad_tile": grad_tile,
               "ms_per_step": {k: round(v, 2) for k, v in med.items()},
               "spread_ms": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
               "bf16_over_bf16x3": round(med["bf16"] / med["bf16x3"], 3),
               "bf16_over_tf32": round(med["bf16"] / med["tf32"], 3),
               "bf16x3_over_tf32": round(med["bf16x3"] / med["tf32"], 3),
               "peak_gib": {k: round(peak(fn), 2) for k, fn in steps.items()},
               "slot_ms": {tp: slots(models[tp], steps[tp]) for tp in ("bf16x3", "bf16")}}
        row["bf16_faster"] = med["bf16"] < med["bf16x3"]
        res.append(row)
        print(json.dumps(row), file=sys.stderr)
        del models, steps, ins, tgt
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "training step (forward, MSE, backward; no VGG), ms per step, median of alternated "
                                "rounds", "gpu": name, "power_limit": limit, "rounds": args.rounds,
                      "steps_per_round": args.steps, "results": res}))


if __name__ == "__main__":
    main()
