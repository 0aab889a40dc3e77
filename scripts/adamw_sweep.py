#!/usr/bin/env python
"""AdamW on the bf16 engine, one GPU (``ShadowEngine(optimizer="adamw")``): what the decoupled weight decay costs
against the same engine running Adam.

* ResNet-18 and VGG-11 on synthetic CIFAR-shaped data at batch ``--batch``; codes svd rank 3 and the dense ``sgd``
  code.  For each (model, code) one engine with ``adam`` and one with ``adamw`` at weight decay ``WD`` (CUDA graph,
  overlap), alternated round by round in one process; the first round warms them.  Step time is the median over rounds
  of CUDA events around ``--steps`` steps.
* The decay kernel (``v2_decay_kernel``, one launch per group) is timed with ``torch.profiler`` in a run of its own for
  each model, svd rank 3.  Its bytes come from shapes: every weight element read and written, 8 bytes each.

The card name and power limit are read in the same run.

    python scripts/adamw_sweep.py --out profiles/adamw_h100_1gpu.json
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from code_stats_sweep import card  # noqa: E402

CODES = [("svd rank 3", dict(code="svd", svd_rank=3)), ("dense", dict(code="sgd"))]
MODELS = ["ResNet18", "VGG11"]
LR, WD = 1e-3, 0.05


def engine(net, kw, optimizer, graph=True):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model(net, 10), 0, 1, seed=1, use_graph=graph, optimizer=optimizer, lr=LR,
                        weight_decay=WD, **kw)


def batch(n, seed=0):
    from atomo_b200.data import SyntheticImageDataset
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=seed).materialize(n)
    return x.cuda(), y.cuda()


def median(v):
    return sorted(v)[len(v) // 2]


def kernel_times(net, batch_n, steps):
    eng = engine(net, CODES[0][1], "adamw", graph=False)
    x, y = batch(batch_n)
    eng.prepare(x, y, warmup=2)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            eng.train_step(x, y)
        torch.cuda.synchronize()
    w = eng.plan.w_total
    ev = [e for e in prof.key_averages() if "v2_decay_kernel" in e.key]
    us = sum(e.device_time_total for e in ev) / steps
    nbytes = 8 * w
    out = {"kernels": sorted(e.key for e in ev), "us_per_step": us, "launches_per_step": sum(e.count for e in ev) / steps,
           "bytes_per_step": nbytes, "GB_per_s": nbytes / (us * 1e-6) / 1e9 if us > 0 else None, "weight_elements": w}
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = {"card": card(), "data": "synthetic CIFAR-shaped", "batch": a.batch, "lr": LR, "weight_decay": WD,
           "step_ms": {}, "kernel_svd": {}}
    x, y = batch(a.batch)
    for net in MODELS:
        for label, ckw in CODES:
            engs = {}
            for opt in ("adam", "adamw"):
                e = engine(net, ckw, opt)
                e.prepare(x, y, warmup=1)
                engs[opt] = e
            times = {k: [] for k in engs}
            for r in range(a.rounds + 1):
                for k, e in engs.items():
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                    for _ in range(a.steps):
                        e.train_step(x, y)
                    ev1.record()
                    torch.cuda.synchronize()
                    assert e.error_code() == 0
                    if r > 0:
                        times[k].append(ev0.elapsed_time(ev1) / a.steps)
            off, on = median(times["adam"]), median(times["adamw"])
            key = "%s %s" % (net, label)
            res["step_ms"][key] = {"adam": off, "adamw": on, "change_pct": 100.0 * (on - off) / off,
                                   "rounds_adam": times["adam"], "rounds_adamw": times["adamw"],
                                   "launches_per_step": {k: e.launches_per_step for k, e in engs.items()}}
            print(key, res["step_ms"][key], flush=True)
            for e in engs.values():
                e.close()
    for net in MODELS:
        res["kernel_svd"][net] = kernel_times(net, a.batch, 10)
        print(net, res["kernel_svd"][net], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
