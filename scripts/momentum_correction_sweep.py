#!/usr/bin/env python
"""Momentum correction (Deep Gradient Compression) against PS momentum for top-k with error feedback, one GPU.

For ResNet-18 and VGG-11 at top-k budgets 1 % and 0.1 %, both arms run top-k with error feedback and momentum 0.9:
``ps`` applies it on the parameter server to the decoded sum, ``mc`` on the workers before sparsifying, with the
momentum of sent entries masked (``momentum_correction=True``).  It times the step (CUDA graph + overlap), alternating
the two arms in one process, then trains ``--train-steps`` fixed-seed steps on the same batch sequence (synthetic
CIFAR shape, batch 128, lr 0.05) and records the loss, ``||e||`` and (``mc``) ``||u||`` curves.  The synthetic set is
memorised quickly, so the curves say nothing about accuracy.  The card name and power limit are read in the same run.

    python scripts/momentum_correction_sweep.py --out profiles/momentum_correction_h100_1gpu.json
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from code_stats_sweep import card  # noqa: E402
from error_feedback_sweep import batches, fin  # noqa: E402

BUDGETS = (0.01, 0.001)
ARMS = ("ps", "mc")


def engine(net, budget, arm):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model(net, 10), 0, 1, code="topk", entry_budget=budget, lr=0.05, momentum=0.9, seed=1,
                        error_feedback=True, momentum_correction=(arm == "mc"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/momentum_correction_h100_1gpu.json)")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--train-steps", type=int, default=100)
    ap.add_argument("--time-steps", type=int, default=100)
    ap.add_argument("--time-reps", type=int, default=5)
    ap.add_argument("--nets", type=str, default="ResNet18,VGG11")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    rec = {"card": card(), "batch": a.batch, "lr": 0.05, "momentum": 0.9, "train_steps": a.train_steps,
           "timing": [], "training": []}
    data = batches(a.train_steps, a.batch)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for net in a.nets.split(","):
        for budget in BUDGETS:
            x, y = data[0]
            engs = {}
            for arm in ARMS:
                engs[arm] = engine(net, budget, arm)
                engs[arm].prepare(x, y, warmup=3)
            times = {arm: [] for arm in ARMS}
            for rep in range(a.time_reps + 1):
                for arm in ARMS:
                    torch.cuda.synchronize()
                    ev0.record()
                    for _ in range(a.time_steps):
                        engs[arm].train_step(x, y)
                    ev1.record()
                    torch.cuda.synchronize()
                    if rep > 0:         # the first round warms both engines
                        times[arm].append(ev0.elapsed_time(ev1) / a.time_steps)
            med = {}
            for arm in ARMS:
                v = sorted(times[arm])
                med[arm] = v[len(v) // 2]
                rec["timing"].append({"net": net, "budget": budget, "arm": arm, "median_ms": round(med[arm], 4),
                                      "step_ms": [round(s, 4) for s in times[arm]],
                                      "launches_per_step": engs[arm].launches_per_step,
                                      "error_code": engs[arm].error_code()})
            print("%-8s %.3f  step ms: ps %.3f  mc %.3f  (%+.3f ms)" % (net, budget, med["ps"], med["mc"],
                                                                         med["mc"] - med["ps"]), flush=True)
            for e in engs.values():
                e.close()
            for arm in ARMS:
                eng = engine(net, budget, arm)
                eng.prepare(*data[0], warmup=0)
                losses, ef_curve, u_curve = [], [], []
                for i, (xb, yb) in enumerate(data):
                    losses.append(eng.train_step(xb, yb)[0].clone())
                    if i % 10 == 0:
                        ef_curve.append(eng.error_feedback_norm()["model"])
                        if arm == "mc":
                            u_curve.append(eng.momentum_correction_norm()["model"])
                torch.cuda.synchronize()
                ls = torch.stack(losses).tolist()
                row = {"net": net, "budget": budget, "arm": arm, "error_code": eng.error_code(),
                       "loss_last10": fin(sum(ls[-10:]) / 10), "loss_curve": [fin(v, 4) for v in ls[::10]],
                       "ef_norm_curve": [fin(v, 4) for v in ef_curve]}
                if arm == "mc":
                    row["mom_norm_curve"] = [fin(v, 4) for v in u_curve]
                eng.close()
                rec["training"].append(row)
                print("%-8s %.3f %s  loss %s  ||e|| %s  ||u|| %s  err %d" % (
                    net, budget, arm, row["loss_last10"], row["ef_norm_curve"][-1],
                    row.get("mom_norm_curve", [None])[-1], row["error_code"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
