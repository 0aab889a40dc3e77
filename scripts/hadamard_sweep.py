#!/usr/bin/env python
"""Randomized-Hadamard rotated quantization against QSGD, TernGrad, fp8 and the dense code on the bf16 engine, one GPU.

For ResNet-18 and VGG-11 it times the step (CUDA graph + overlap) of ``hadamard`` at 2 / 4 / 8 bits with bucket 512
and at 4 bits with buckets 64 and 4096, each with error feedback off and on, then ``qsgd`` levels 2 and 4, ``terngrad``
and ``fp8`` at bucket 512 and the uncompressed ``sgd`` engine, alternating all engines of a net in one process (median
of the rounds), and reads each engine's device-side encode time per step (``phase_stats()``).  Then, with fixed seeds,
it trains ``--train-steps`` steps of each coded configuration on the same batch sequence (synthetic CIFAR shape, batch
128, lr 0.05, momentum 0.9) and records the loss curve, the final ``||e||``, whether the loss stayed finite, and the
whole-model ``rel_var`` and push MiB of ``code_stats()``.  Beside the measured ``rel_var`` it records the oracle's
(``codings/hadamard.py``, fp64 on the CPU) ``rel_var`` of one fp32 backward at initialisation.  The card name and
power limit are read in the same run.

    python scripts/hadamard_sweep.py --out profiles/hadamard_h100_1gpu.json
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

HAD = [(2, 512), (4, 512), (8, 512), (4, 64), (4, 4096)]
CONFS = [("hadamard", p, ef) for p in HAD for ef in (False, True)] + \
    [("qsgd", (2, 512), False), ("qsgd", (4, 512), False), ("terngrad", (1, 512), False), ("fp8", (0, 512), False),
     ("sgd", None, False)]


def engine(net, code, param, ef, stats=False):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    kw = {}
    if code in ("hadamard", "qsgd", "terngrad"):
        kw = {"quantization_level": param[0], "bucket_size": param[1]}
    elif code == "fp8":
        kw = {"bucket_size": param[1]}
    return ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=0.05, momentum=0.9, seed=1, error_feedback=ef,
                        code_stats=stats and code != "sgd", **kw)


def cpu_estimate(net, x, y):
    """The oracle's rel_var of one fp32 backward of the initial model, per bits at bucket 512."""
    from atomo_b200.codings.hadamard import Hadamard
    from atomo_b200.models import build_model
    torch.manual_seed(0)
    m = build_model(net, 10).cuda()
    torch.nn.functional.cross_entropy(m(x.cuda().float()), y.cuda()).backward()
    grads = []
    for p in m.parameters():
        if p.dim() >= 2:
            g = p.grad.detach().float().cpu()
            grads.append(g.permute(0, 2, 3, 1).reshape(-1) if g.dim() == 4 else g.reshape(-1))
    out = {}
    for bits in (2, 4, 8):
        c = Hadamard(bits, 512, seed=1)
        mse = sum(c.expected_error_sq(g, unit=i, step=1) for i, g in enumerate(grads))
        gsq = sum(float(g.bfloat16().double().square().sum()) for g in grads)
        out[str(bits)] = mse / gsq
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/hadamard_h100_1gpu.json)")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--train-steps", type=int, default=100)
    ap.add_argument("--time-steps", type=int, default=100)
    ap.add_argument("--time-reps", type=int, default=5)
    ap.add_argument("--nets", type=str, default="ResNet18,VGG11")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    rec = {"card": card(), "batch": a.batch, "lr": 0.05, "momentum": 0.9, "train_steps": a.train_steps,
           "timing": [], "training": [], "cpu_estimate_rel_var_at_init": {}}
    data = batches(a.train_steps, a.batch)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for net in a.nets.split(","):
        rec["cpu_estimate_rel_var_at_init"][net] = est = cpu_estimate(net, *data[0])
        print("%-8s CPU oracle rel_var at init (bucket 512): %s" % (net, est), flush=True)
        x, y = data[0]
        engs = {}
        for c in CONFS:
            engs[c] = engine(net, *c)
            engs[c].prepare(x, y, warmup=3)
        times = {c: [] for c in CONFS}
        enc = {c: [] for c in CONFS}
        for rep in range(a.time_reps + 1):
            for c in CONFS:
                torch.cuda.synchronize()
                engs[c].phase_stats(reset=True)
                ev0.record()
                for _ in range(a.time_steps):
                    engs[c].train_step(x, y)
                ev1.record()
                torch.cuda.synchronize()
                ph = engs[c].phase_stats(reset=True)
                if rep > 0:         # the first round warms every engine
                    times[c].append(ev0.elapsed_time(ev1) / a.time_steps)
                    enc[c].append(ph["encode_us"])
        for c in CONFS:
            v, e = sorted(times[c]), sorted(enc[c])
            t = {"net": net, "code": c[0], "param": c[1], "error_feedback": c[2],
                 "median_ms": round(v[len(v) // 2], 4), "step_ms": [round(s, 4) for s in times[c]],
                 "encode_us": round(e[len(e) // 2], 2), "error_code": engs[c].error_code()}
            rec["timing"].append(t)
            print("%-8s %-8s %-10s ef=%d  step ms %.3f  encode us %.1f" % (net, c[0], c[1], c[2], t["median_ms"],
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
                   "rel_var": fin(st["rel_var"], 6), "push_mib": round(st["bytes"] / 2 ** 20, 4),
                   "atoms": round(st["atoms"], 1)}
            if ef:
                row["ef_norm"] = fin(eng.error_feedback_norm()["model"], 4)
                row["ef_norm_curve"] = [fin(v, 4) for v in ef_curve]
            eng.close()
            rec["training"].append(row)
            print("%-8s %-8s %-10s ef=%d  loss %s  rel_var %s  push %.3f MiB  ||e|| %s  err %d" % (
                net, code, param, ef, row["loss_last10"], row["rel_var"], row["push_mib"], row.get("ef_norm"),
                row["error_code"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
