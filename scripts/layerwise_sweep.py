#!/usr/bin/env python
"""LARS and LAMB on the bf16 engine, one GPU (``ShadowEngine(optimizer='lars' | 'lamb')``): what the layer-wise step
costs against the optimizer it extends.

* ResNet-18 on synthetic CIFAR-shaped data at micro-batch ``--micro``, codes svd rank 3 and the dense ``sgd`` code:
  SGD against LARS and Adam against LAMB, at ``--accumulate-steps`` 1 and 8.  One engine per configuration (CUDA
  graph, overlap), the four optimizers of a (code, N) alternated round by round in one process; the first round warms
  them.  Step time is the median over rounds of CUDA events around ``--steps`` steps.
* Phase 2 (``v2_layerwise_kernel``) is timed with ``torch.profiler`` in a run of its own: its device time per step
  summed over the backward groups.  Its bytes come from shapes: per weight element it reads master, the direction and
  (LARS) the momentum, writes master and (LARS) the momentum, and stores 2 bytes of bf16 weight.
* A short loss curve of LAMB and LARS at a global batch of 1024 (micro-batch 128, N = 8) on the synthetic set: it is
  synthetic data, so it says that training moves, not how well it generalises.

The card name and power limit are read in the same run.

    python scripts/layerwise_sweep.py --out profiles/layerwise_h100_1gpu.json
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from code_stats_sweep import card  # noqa: E402

OPTS = {"sgd": dict(optimizer="sgd", lr=0.05, momentum=0.9, weight_decay=5e-4),
        "lars": dict(optimizer="lars", lr=2.0, momentum=0.9, weight_decay=5e-4, trust_coefficient=0.001),
        "adam": dict(optimizer="adam", lr=1e-3, weight_decay=0.0),
        "lamb": dict(optimizer="lamb", lr=5e-3, weight_decay=0.01)}
CODES = [("svd", {"svd_rank": 3}, "svd rank 3"), ("sgd", {}, "dense")]


def engine(code, kw, opt, n, graph=True):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model("ResNet18", 10), 0, 1, code=code, seed=1, use_graph=graph, accumulate_steps=n,
                        **dict(kw, **OPTS[opt]))


def batch(n, seed=0):
    from atomo_b200.data import SyntheticImageDataset
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=seed).materialize(n)
    return x.cuda(), y.cuda()


def median(v):
    return sorted(v)[len(v) // 2]


def phase2_bytes(eng):
    w = eng.plan.w_total
    per = (4 * 3 + 4 * 2 + 2) if eng.optimizer == "lars" else (4 * 2 + 4 + 2)
    return w * per


def phase2_us(code, kw, opt, micro, steps):
    eng = engine(code, kw, opt, 1, graph=False)
    x, y = batch(micro)
    eng.prepare(x, y, warmup=2)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            eng.train_step(x, y)
        torch.cuda.synchronize()
    tot = sum(e.device_time_total for e in prof.key_averages() if "v2_layerwise_kernel" in e.key)
    n = sum(e.count for e in prof.key_averages() if "v2_layerwise_kernel" in e.key)
    b = phase2_bytes(eng)
    eng.close()
    us = tot / steps
    return {"us_per_step": us, "launches_per_step": n / steps, "bytes_per_step": b,
            "GB_per_s": b / (us * 1e-6) / 1e9 if us > 0 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--micro", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--curve-steps", type=int, default=30)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = {"card": card(), "model": "ResNet18", "data": "synthetic CIFAR-shaped", "micro_batch": a.micro,
           "step_ms": {}, "phase2": {}, "loss_curve_synthetic_batch1024": {}}
    for code, kw, label in CODES:
        for n in (1, 8):
            x, y = batch(n * a.micro)
            engs = {}
            for opt in OPTS:
                e = engine(code, kw, opt, n)
                e.prepare(x, y, warmup=1)
                engs[opt] = e
            times = {opt: [] for opt in OPTS}
            for r in range(a.rounds + 1):
                for opt, e in engs.items():
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                    for _ in range(a.steps):
                        e.train_step(x, y)
                    ev1.record()
                    torch.cuda.synchronize()
                    assert e.error_code() == 0
                    if r > 0:
                        times[opt].append(ev0.elapsed_time(ev1) / a.steps)
            for opt, e in engs.items():
                res["step_ms"]["%s N=%d %s" % (label, n, opt)] = median(times[opt])
                e.close()
            print(label, n, {o: round(median(t), 3) for o, t in times.items()}, flush=True)
        for opt in ("lars", "lamb"):
            res["phase2"]["%s %s" % (label, opt)] = phase2_us(code, kw, opt, a.micro, 10)
            print(label, opt, res["phase2"]["%s %s" % (label, opt)], flush=True)
    for opt in ("lars", "lamb"):
        e = engine("svd", {"svd_rank": 3}, opt, 8)
        x, y = batch(8 * a.micro)
        e.prepare(x, y, warmup=0)
        curve = []
        for s in range(a.curve_steps):
            x, y = batch(8 * a.micro, seed=s % 4)
            curve.append(float(e.train_step(x, y)[0]))
        torch.cuda.synchronize()
        assert e.error_code() == 0
        res["loss_curve_synthetic_batch1024"]["svd rank 3 " + opt] = curve
        e.close()
        print(opt, "loss", curve[0], "->", curve[-1], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res)[:2000])


if __name__ == "__main__":
    main()
