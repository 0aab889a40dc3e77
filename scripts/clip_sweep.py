#!/usr/bin/env python
"""Gradient-norm clipping on the bf16 engine, one GPU (``ShadowEngine(clip_grad_norm=MAX)``): what the deferred,
whole-model step costs against the same engine without clipping.

* ResNet-18 and VGG-11 on synthetic CIFAR-shaped data at batch ``--batch``; codes svd rank 3, the dense ``sgd`` code
  and top-k with error feedback; optimizers momentum-SGD, Adam and LAMB.  For each (model, code, optimizer) one
  engine with clipping off and one with it on (CUDA graph, overlap), alternated round by round in one process; the
  first round warms them.  Step time is the median over rounds of CUDA events around ``--steps`` steps.
* The gather (phase 1) and clip (phase 2) kernels are timed with ``torch.profiler`` in a run of their own, ResNet-18,
  svd rank 3, momentum-SGD.  Their bytes come from shapes.  Gather writes g, 4 bytes per weight and vector element,
  on top of the work the plain PS kernel does.  The clip launch reads g, master and the momentum, writes master and
  the momentum, and stores 2 bytes of bf16 weight per weight element: 22 bytes.  It does 4 + 4 + 4 reads and
  4 + 4 + 4 writes per vector element.
* Arithmetic only, not measured: deferring the step adds about 8 bytes per weight element (g written, then read).

The card name and power limit are read in the same run.

    python scripts/clip_sweep.py --out profiles/clip_h100_1gpu.json
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from code_stats_sweep import card  # noqa: E402

OPTS = {"momentum": dict(optimizer="sgd", lr=0.05, momentum=0.9, weight_decay=5e-4),
        "adam": dict(optimizer="adam", lr=1e-3),
        "lamb": dict(optimizer="lamb", lr=5e-3, weight_decay=0.01)}
CODES = [("svd rank 3", dict(code="svd", svd_rank=3)), ("dense", dict(code="sgd")),
         ("topk+EF", dict(code="topk", entry_budget=0.01, error_feedback=True))]
MODELS = ["ResNet18", "VGG11"]
MAX_NORM = 1.0


def engine(net, kw, clip, graph=True):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model(net, 10), 0, 1, seed=1, use_graph=graph, clip_grad_norm=clip, **kw)


def batch(n, seed=0):
    from atomo_b200.data import SyntheticImageDataset
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=seed).materialize(n)
    return x.cuda(), y.cuda()


def median(v):
    return sorted(v)[len(v) // 2]


def kernel_times(batch_n, steps):
    eng = engine("ResNet18", dict(CODES[0][1], **OPTS["momentum"]), MAX_NORM, graph=False)
    x, y = batch(batch_n)
    eng.prepare(x, y, warmup=2)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            eng.train_step(x, y)
        torch.cuda.synchronize()
    w, v = eng.plan.w_total, eng.plan.v_total
    out = {}
    for name, key, nbytes in (("gather", "gather_kernel", 4 * (w + v)), ("clip", "v2_clip_kernel", 22 * w + 24 * v)):
        ev = [e for e in prof.key_averages() if key in e.key]
        us = sum(e.device_time_total for e in ev) / steps
        out[name] = {"kernels": sorted(e.key for e in ev), "us_per_step": us,
                     "launches_per_step": sum(e.count for e in ev) / steps, "bytes_per_step": nbytes,
                     "GB_per_s": nbytes / (us * 1e-6) / 1e9 if us > 0 else None}
    out["weight_elements"], out["vector_elements"] = w, v
    out["deferral_bytes_arithmetic"] = 8 * w
    out["deferral_us_at_3.35TB_s_arithmetic"] = 8 * w / 3.35e12 * 1e6
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = {"card": card(), "data": "synthetic CIFAR-shaped", "batch": a.batch, "clip_grad_norm": MAX_NORM,
           "step_ms": {}, "kernels_resnet18_svd_momentum": {}}
    x, y = batch(a.batch)
    for net in MODELS:
        for label, ckw in CODES:
            for opt, okw in OPTS.items():
                engs = {}
                for clip in (0.0, MAX_NORM):
                    e = engine(net, dict(ckw, **okw), clip)
                    e.prepare(x, y, warmup=1)
                    engs["on" if clip else "off"] = e
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
                off, on = median(times["off"]), median(times["on"])
                total, coef = engs["on"].grad_norm()
                key = "%s %s %s" % (net, label, opt)
                res["step_ms"][key] = {"off": off, "on": on, "change_pct": 100.0 * (on - off) / off,
                                       "last_grad_norm": total, "last_clip_coef": coef}
                print(key, res["step_ms"][key], flush=True)
                for e in engs.values():
                    e.close()
    res["kernels_resnet18_svd_momentum"] = kernel_times(a.batch, 10)
    print(res["kernels_resnet18_svd_momentum"], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
