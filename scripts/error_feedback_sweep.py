#!/usr/bin/env python
"""Error feedback on the bf16 engine, one GPU (``ShadowEngine(error_feedback=True)``): what it costs per step and what
it does to the training loss, on synthetic CIFAR-shaped data.

For ResNet-18 and VGG-11 it times the step with error feedback off and on, alternating the two engines in the same
process, for each code below.  Then, for each code and with fixed seeds, it trains ``--train-steps`` steps on the same
batch sequence with error feedback off and on and records the loss (mean of the last 10 steps) and the final
``||e||``.  The card name and power limit are read in the same run.

    python scripts/error_feedback_sweep.py --out profiles/error_feedback_h100_1gpu.json
"""
import argparse
import json
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from code_stats_sweep import card  # noqa: E402

CONFIGS = [("svd", {"svd_rank": 1, "random_sample": False}, "svd rank 1, top-k"),
           ("svd", {"svd_rank": 3}, "svd rank 3, sampled"),
           ("entrywise", {"entry_budget": 0.01}, "entry-wise 1 %"),
           ("qsgd", {"quantization_level": 2}, "QSGD level 2")]


def fin(v, nd=5):
    """JSON has no NaN / Inf: a diverged run records null"""
    return round(v, nd) if math.isfinite(v) else None


def engine(net, code, kw, ef, batch, lr=0.05):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=lr, momentum=0.9, seed=1, error_feedback=ef, **kw)


def batches(n, batch, seed=0):
    from atomo_b200.data import SyntheticImageDataset
    ds = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=seed)
    x, y = ds.materialize(4096)
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        i = torch.randint(0, x.shape[0], (batch,), generator=g)
        out.append((x[i].cuda(), y[i].cuda()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/error_feedback_h100_1gpu.json)")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--train-steps", type=int, default=100)
    ap.add_argument("--time-steps", type=int, default=100)
    ap.add_argument("--time-reps", type=int, default=5)
    ap.add_argument("--nets", type=str, default="ResNet18,VGG11")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    rec = {"card": card(), "batch": a.batch, "train_steps": a.train_steps, "timing": [], "training": []}
    data = batches(a.train_steps, a.batch)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for net in a.nets.split(","):
        for code, kw, label in CONFIGS:
            # step time, error feedback off / on alternated in one process (CUDA graph + overlap)
            x, y = data[0]
            engs = {}
            for ef in (False, True):
                engs[ef] = engine(net, code, kw, ef, a.batch)
                engs[ef].prepare(x, y, warmup=3)
            times = {False: [], True: []}
            for rep in range(a.time_reps + 1):
                for ef in (False, True):
                    torch.cuda.synchronize()
                    ev0.record()
                    for _ in range(a.time_steps):
                        engs[ef].train_step(x, y)
                    ev1.record()
                    torch.cuda.synchronize()
                    if rep > 0:         # the first round warms both engines
                        times[ef].append(ev0.elapsed_time(ev1) / a.time_steps)
            errs = {ef: engs[ef].error_code() for ef in (False, True)}
            for e in engs.values():
                e.close()
            med = {ef: sorted(v)[len(v) // 2] for ef, v in times.items()}
            t = {"net": net, "code": label, "median_ms_off": round(med[False], 4), "median_ms_on": round(med[True], 4),
                 "overhead_pct": round(100.0 * (med[True] / med[False] - 1.0), 2),
                 "step_ms_off": [round(v, 4) for v in times[False]], "step_ms_on": [round(v, 4) for v in times[True]],
                 "error_code_off": errs[False], "error_code_on": errs[True]}
            rec["timing"].append(t)
            print("%-8s %-22s step ms off %.3f on %.3f (%+.2f%%)" % (net, label, med[False], med[True],
                                                                      t["overhead_pct"]), flush=True)
            # training loss over the same seeded batch sequence, off and on
            row = {"net": net, "code": label, **kw}
            for ef in (False, True):
                eng = engine(net, code, kw, ef, a.batch)
                eng.prepare(*data[0], warmup=0)
                losses, ef_curve = [], []
                for i, (x, y) in enumerate(data):
                    losses.append(eng.train_step(x, y)[0].clone())
                    if ef and i % 10 == 0:
                        ef_curve.append(eng.error_feedback_norm()["model"])
                torch.cuda.synchronize()
                ls = torch.stack(losses).tolist()
                key = "on" if ef else "off"
                # a non-zero code is recorded, not hidden: 8 = a non-finite Gram matrix (the run diverged)
                row["error_code_" + key] = eng.error_code()
                row["loss_" + key] = fin(sum(ls[-10:]) / 10)
                row["loss_curve_" + key] = [fin(v, 4) for v in ls[::10]]
                if ef:
                    row["ef_norm"] = fin(eng.error_feedback_norm()["model"], 4)
                    row["ef_norm_curve"] = [fin(v, 4) for v in ef_curve]
                eng.close()
            rec["training"].append(row)
            print("%-8s %-22s loss after %d steps: off %s on %s, ||e|| %s, error codes %d / %d" % (
                net, label, a.train_steps, row["loss_off"], row["loss_on"], row["ef_norm"], row["error_code_off"],
                row["error_code_on"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
