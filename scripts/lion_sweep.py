#!/usr/bin/env python
"""Lion on the bf16 engine, one GPU (``ShadowEngine(optimizer="lion")``): step time, parameter-server work and owner
state against momentum-SGD, Adam and AdamW on the same engine.

* ResNet-18 and VGG-11 on synthetic CIFAR-shaped data at batch ``--batch``; codes svd rank 3, dense, top-k with error
  feedback and fp8.  For each (model, code) one engine per optimizer (momentum-SGD, Adam, AdamW, Lion, Lion with
  weight decay; CUDA graph, overlap), alternated round by round in one process; the first round warms them.  Step time
  is the median over rounds of CUDA events around ``--steps`` steps; ``ps_work_us`` is the median of
  ``phase_stats()['ps_work_us']`` over the same rounds (device globaltimer stamps inside the PS kernels).
* Owner state: the fp32 bytes the owner keeps per weight and vector element (master, mom, sq, sqmax; vparams, vmom,
  vsq, vsqmax), counted from the allocated tensors.
* A short loss curve per optimizer (ResNet-18, svd rank 3, fresh synthetic batches) as a sanity check only: it makes
  no accuracy claim.

The card name and power limit are read in the same run.

    python scripts/lion_sweep.py --out profiles/lion_h100_1gpu.json
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from code_stats_sweep import card  # noqa: E402

CODES = [("svd rank 3", dict(code="svd", svd_rank=3)), ("dense", dict(code="sgd")),
         ("topk + EF", dict(code="topk", entry_budget=0.05, error_feedback=True)), ("fp8", dict(code="fp8"))]
MODELS = ["ResNet18", "VGG11"]
OPTS = {
    "sgd-momentum": dict(optimizer="sgd", lr=0.05, momentum=0.9),
    "adam": dict(optimizer="adam", lr=1e-3),
    "adamw": dict(optimizer="adamw", lr=1e-3, weight_decay=0.05),
    "lion": dict(optimizer="lion", lr=1e-4),
    "lion wd": dict(optimizer="lion", lr=1e-4, weight_decay=0.5),
}


def engine(net, kw, okw, graph=True):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model(net, 10), 0, 1, seed=1, use_graph=graph, **okw, **kw)


def batch(n, seed=0):
    from atomo_b200.data import SyntheticImageDataset
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=seed).materialize(n)
    return x.cuda(), y.cuda()


def median(v):
    return sorted(v)[len(v) // 2]


def state_bytes(e):
    w = sum(t.numel() * 4 for t in (e.master, e.mom, e.sq, e.sqmax) if t is not None)
    v = sum(t.numel() * 4 for t in (e.vparams, e.vmom, e.vsq, e.vsqmax) if t is not None)
    return {"weight_bytes": w, "vector_bytes": v, "bytes_per_weight_element": w / e.plan.w_total}


def loss_curve(okw, batch_n, steps, every):
    e = engine("ResNet18", CODES[0][1], okw)
    x, y = batch(batch_n, 1000)
    e.prepare(x, y, warmup=0)
    out = []
    for s in range(steps):
        x, y = batch(batch_n, 1000 + s % 8)
        loss = e.train_step(x, y)
        if (s + 1) % every == 0:
            torch.cuda.synchronize()
            out.append(float(loss[0]))
    assert e.error_code() == 0
    e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--curve-steps", type=int, default=80)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = {"card": card(), "data": "synthetic CIFAR-shaped", "batch": a.batch, "optimizers": OPTS, "step_ms": {},
           "ps_work_us": {}, "owner_state": {}, "loss_curve_resnet18_svd": {}}
    x, y = batch(a.batch)
    for net in MODELS:
        for label, ckw in CODES:
            engs = {}
            for k, okw in OPTS.items():
                e = engine(net, ckw, okw)
                e.prepare(x, y, warmup=1)
                engs[k] = e
            times, ps = {k: [] for k in engs}, {k: [] for k in engs}
            for r in range(a.rounds + 1):
                for k, e in engs.items():
                    e.phase_stats(reset=True)
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                    for _ in range(a.steps):
                        e.train_step(x, y)
                    ev1.record()
                    torch.cuda.synchronize()
                    assert e.error_code() == 0
                    st = e.phase_stats(reset=True)
                    if r > 0:
                        times[k].append(ev0.elapsed_time(ev1) / a.steps)
                        ps[k].append(st["ps_work_us"])
            key = "%s %s" % (net, label)
            res["step_ms"][key] = {k: {"median": median(v), "rounds": v} for k, v in times.items()}
            res["ps_work_us"][key] = {k: {"median": median(v), "rounds": v} for k, v in ps.items()}
            res["owner_state"][key] = {k: state_bytes(e) for k, e in engs.items()}
            print(key, {k: round(median(v), 3) for k, v in times.items()},
                  {k: round(median(v), 1) for k, v in ps.items()}, flush=True)
            for e in engs.values():
                e.close()
    for k, okw in OPTS.items():
        res["loss_curve_resnet18_svd"][k] = loss_curve(okw, a.batch, a.curve_steps, 10)
        print("loss", k, res["loss_curve_resnet18_svd"][k], flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
