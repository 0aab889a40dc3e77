#!/usr/bin/env python
"""PowerSGD against the other contractive codes on the bf16 engine, one GPU, with error feedback off and on.

For ResNet-18 and VGG-11 it times the step (CUDA graph + overlap) of ``powersgd`` at r = 1 / 2 / 4 with error feedback
off and on, beside top-k 1 %, sign (bucket 512) and spectral top-k (``svd`` rank 1, ``random_sample=False``), all
three with error feedback, and the uncompressed ``sgd`` engine.  All engines of a net alternate in one process (median
of the rounds); the device-side encode time of each engine (``phase_stats()['encode_us']``, first encode CTA in to last
push published, summed over the backward groups) is read over the same rounds.  Then, with fixed seeds, it trains
``--train-steps`` steps of each coded configuration on the same batch sequence (synthetic CIFAR shape, batch 128,
lr 0.05, momentum 0.9) and records the loss curve, the ``||e||`` curve, whether the loss stayed finite, and the
whole-model ``rel_var`` and push MB of ``code_stats()``.  The card name and power limit are read in the same run.

    python scripts/powersgd_sweep.py --out profiles/powersgd_h100_1gpu.json
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
from error_feedback_sweep import batches, fin  # noqa: E402

CONFS = [("powersgd", r, ef) for r in (1, 2, 4) for ef in (False, True)] + \
    [("topk", 0.01, True), ("sign", 512, True), ("svd", 1, True), ("sgd", None, False)]


def engine(net, code, param, ef, stats=False):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    kw = {"powersgd": {"svd_rank": param}, "topk": {"entry_budget": param}, "sign": {"bucket_size": param},
          "svd": {"svd_rank": param, "random_sample": False}}.get(code, {})
    return ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=0.05, momentum=0.9, seed=1, error_feedback=ef,
                        code_stats=stats and code != "sgd", **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/powersgd_h100_1gpu.json)")
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
        x, y = data[0]
        engs = {}
        for c in CONFS:
            engs[c] = engine(net, *c)
            engs[c].prepare(x, y, warmup=3)
        times = {c: [] for c in CONFS}
        for rep in range(a.time_reps + 1):
            for c in CONFS:
                torch.cuda.synchronize()
                if rep == 1:
                    engs[c].phase_stats(reset=True)
                ev0.record()
                for _ in range(a.time_steps):
                    engs[c].train_step(x, y)
                ev1.record()
                torch.cuda.synchronize()
                if rep > 0:         # the first round warms every engine
                    times[c].append(ev0.elapsed_time(ev1) / a.time_steps)
        for c in CONFS:
            v = sorted(times[c])
            t = {"net": net, "code": c[0], "param": c[1], "error_feedback": c[2],
                 "median_ms": round(v[len(v) // 2], 4), "step_ms": [round(s, 4) for s in times[c]],
                 "encode_us": round(engs[c].phase_stats()["encode_us"], 1), "error_code": engs[c].error_code()}
            rec["timing"].append(t)
            print("%-8s %-8s %-5s ef=%d  step ms %.3f  encode us %.1f" % (net, c[0], c[1], c[2], t["median_ms"],
                                                                        t["encode_us"]), flush=True)
        for e in engs.values():
            e.close()
        for code, param, ef in CONFS:
            if code == "sgd":
                continue
            eng = engine(net, code, param, ef, stats=True)
            eng.prepare(*data[0], warmup=0)
            eng.code_stats(reset=True)
            losses, ef_curve = [], []
            for i, (xb, yb) in enumerate(data):
                losses.append(eng.train_step(xb, yb)[0].clone())
                if ef and i % 10 == 0:
                    ef_curve.append(eng.error_feedback_norm()["model"])
            torch.cuda.synchronize()
            st = eng.code_stats()["model"]
            ls = torch.stack(losses).tolist()
            row = {"net": net, "code": code, "param": param, "error_feedback": ef,
                   "error_code": eng.error_code(), "loss_finite": all(math.isfinite(v) for v in ls),
                   "loss_last10": fin(sum(ls[-10:]) / 10), "loss_curve": [fin(v, 4) for v in ls[::10]],
                   "rel_var": fin(st["rel_var"], 6), "push_mb": round(st["bytes"] / 2 ** 20, 4),
                   "atoms": round(st["atoms"], 1)}
            if ef:
                row["ef_norm"] = fin(eng.error_feedback_norm()["model"], 4)
                row["ef_norm_curve"] = [fin(v, 4) for v in ef_curve]
            eng.close()
            rec["training"].append(row)
            print("%-8s %-8s %-5s ef=%d  loss %s  rel_var %s  push %.3f MB  ||e|| %s  err %d" % (
                net, code, param, ef, row["loss_last10"], row["rel_var"], row["push_mb"], row.get("ef_norm"),
                row["error_code"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
