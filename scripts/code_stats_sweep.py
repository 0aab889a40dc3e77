#!/usr/bin/env python
"""Estimator statistics of the bf16 engine on one GPU (``ShadowEngine(code_stats=True)``): the GPU counterpart of
``variance_study.py``, measured by the engine's own kernels on its own units (block decomposition, bf16 gradient,
physical element order, warm-started Jacobi basis) during training on synthetic CIFAR-shaped data.

For ResNet-18 and VGG-11 and every code setting below it trains ``--warmup`` steps, resets the statistics, trains
``--steps`` more and records per layer and for the whole model the mean ``rel_var`` = E||g_hat - g||^2 / ||g||^2,
expected / realized atoms and realized push bytes.  Then it times the ResNet-18 headline (svd rank 3) with and without
``code_stats``, alternating the two engines in the same process, and records the card name and power limit.

    python scripts/code_stats_sweep.py --out profiles/code_stats_h100_1gpu.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = ([("svd", {"svd_rank": r}) for r in (1, 2, 3, 4, 8)] +
           [("entrywise", {"entry_budget": b}) for b in (0.01, 0.05, 0.25)] +
           [("qsgd", {"quantization_level": q}) for q in (2, 4, 8)] +
           [("terngrad", {"quantization_level": 1})])


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in out.split(",")]
    except Exception as e:          # the record says so instead of guessing
        info["power_limit"] = "unknown (%s)" % type(e).__name__
    return info


def engine(net, code, kw, stats, batch):
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=0).materialize(batch)
    eng = ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=0.05, momentum=0.9, seed=1, code_stats=stats, **kw)
    eng.prepare(x.pin_memory(), y.pin_memory(), warmup=3)
    return eng, x.cuda(), y.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/code_stats_h100_1gpu.json)")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--time-steps", type=int, default=100)
    ap.add_argument("--time-reps", type=int, default=5)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    rec = {"card": card(), "batch": a.batch, "warmup": a.warmup, "steps": a.steps, "runs": []}
    for net in ("ResNet18", "VGG11"):
        for code, kw in CONFIGS:
            eng, x, y = engine(net, code, kw, True, a.batch)
            for _ in range(a.warmup):
                eng.train_step(x, y)
            eng.code_stats(reset=True)
            for _ in range(a.steps):
                eng.train_step(x, y)
            st = eng.code_stats(reset=True)
            assert eng.error_code() == 0
            eng.close()
            rnd = lambda t: {k: (round(v, 6) if isinstance(v, float) else v) for k, v in t.items()}
            rec["runs"].append({"net": net, "code": code, **kw, "steps": st["steps"], "model": rnd(st["model"]),
                                "layers": {n: rnd(t) for n, t in st["tensors"].items()}})
            m = st["model"]
            print("%-8s %-9s %-28s rel_var %9.4f  atoms %10.1f / %10.1f  MB %8.3f" % (
                net, code, kw, m["rel_var"], m["atoms"], m["exp_atoms"], m["bytes"] / 2 ** 20), flush=True)
    # step time of the headline with and without the statistics, alternating the two engines
    engs = {False: engine("ResNet18", "svd", {"svd_rank": 3}, False, a.batch),
            True: engine("ResNet18", "svd", {"svd_rank": 3}, True, a.batch)}
    times = {False: [], True: []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rep in range(a.time_reps + 1):
        for on in (False, True):
            eng, x, y = engs[on]
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(a.time_steps):
                eng.train_step(x, y)
            ev1.record()
            torch.cuda.synchronize()
            if rep > 0:             # the first round warms both engines
                times[on].append(ev0.elapsed_time(ev1) / a.time_steps)
    for eng, _, _ in engs.values():
        assert eng.error_code() == 0
        eng.close()
    med = {on: sorted(v)[len(v) // 2] for on, v in times.items()}
    rec["timing"] = {"config": "ResNet18 svd rank 3, batch %d, CUDA graph + overlap" % a.batch,
                     "step_ms_off": [round(t, 4) for t in times[False]], "step_ms_on": [round(t, 4) for t in times[True]],
                     "median_ms_off": round(med[False], 4), "median_ms_on": round(med[True], 4),
                     "overhead_pct": round(100.0 * (med[True] / med[False] - 1.0), 2)}
    print("step ms off %.3f on %.3f (%+.2f%%)" % (med[False], med[True], rec["timing"]["overhead_pct"]))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
