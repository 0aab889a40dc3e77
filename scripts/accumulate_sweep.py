#!/usr/bin/env python
"""Gradient accumulation on the bf16 engine, one GPU (``ShadowEngine(accumulate_steps=N)``): device time and push
bytes per sample, the cost of the accumulate passes, and the peak memory it saves.

* For ResNet-18 on synthetic CIFAR-shaped data at micro-batch ``--micro`` and each code below, one engine per
  ``N`` in ``--ns`` (CUDA graph, overlap), the engines alternated round by round in one process; the first round warms
  them.  Device time per sample is the median step time over ``N * micro``.
* Push bytes per step come from ``code_stats()`` (realized bytes, one step at N = 1); per sample they fall as
  ``1 / (N * micro)``.  On one GPU nothing crosses a link, so these are bytes, not a measured saving.
* The accumulate passes are timed on their own with CUDA events over ``--kernel-reps`` launches each, over every
  backward group of ResNet-18 at once (the add of a micro-batch before the last, and the fold of the last), with
  the bytes they must move per launch.
* Peak allocated memory of ResNet-50 (CIFAR) at a global batch of ``--mem-batch``: N = 1 against N = ``--mem-n``.

The card name and power limit are read in the same run.

    python scripts/accumulate_sweep.py --out profiles/accumulate_h100_1gpu.json
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

CONFIGS = [("svd", {"svd_rank": 3}, "svd rank 3"),
           ("topk", {"entry_budget": 0.01, "error_feedback": True}, "top-k 1 % + EF"),
           ("fp8", {}, "fp8")]


def engine(net, code, kw, n, graph=True, **extra):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=0.05, momentum=0.9, seed=1, use_graph=graph,
                        accumulate_steps=n, **dict(kw, **extra))


def batch(n, seed=0):
    from atomo_b200.data import SyntheticImageDataset
    x, y = SyntheticImageDataset((3, 32, 32), 10, 4096, seed=seed).materialize(n)
    return x.cuda(), y.cuda()


def median(v):
    return sorted(v)[len(v) // 2]


def time_passes(micro, reps):
    """Both passes over all of ResNet-18's groups, on the gradient buffers an eager step left behind."""
    eng = engine("ResNet18", "svd", {"svd_rank": 3}, 2, graph=False, overlap=False)
    x, y = batch(2 * micro)
    eng.prepare(x, y, warmup=1)
    eng.train_step(x, y)
    torch.cuda.synchronize()
    C, pl = eng.C, eng.plan
    nw, nv = sum(c for _, c in eng.ef_range), sum(c for _, c in eng.vec_range)
    w_elems, v_elems = sum(q.numel for q in pl.params if q.is_w), sum(q.numel for q in pl.params if not q.is_w)
    args = (eng.t_ef_chunks.data_ptr(), nw, eng.t_vec_chunks.data_ptr(), nv, eng.t_gptr.data_ptr(),
            eng.acc.data_ptr(), eng.vacc.data_ptr(), eng.vgrads.data_ptr())
    launches = {"add": lambda: C.v2_accum_add(*args, False), "add_first": lambda: C.v2_accum_add(*args, True),
                "fold": lambda: C.v2_accum_fold(*args, eng.inv_n, 0)}
    # bytes each pass must move: bf16 gradient, fp32 accumulator, fp32 vectors
    need = {"add": 10 * w_elems + 12 * v_elems, "add_first": 6 * w_elems + 8 * v_elems,
            "fold": 12 * w_elems + 16 * v_elems}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {"weight_elements": w_elems, "vector_elements": v_elems, "chunks": nw + nv}
    for name, fn in launches.items():
        for _ in range(20):
            fn()
        samples = []
        for _ in range(5):
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(reps):
                fn()
            ev1.record()
            torch.cuda.synchronize()
            samples.append(ev0.elapsed_time(ev1) * 1e3 / reps)
        us = median(samples)
        out[name] = {"us": round(us, 2), "us_samples": [round(v, 2) for v in samples], "bytes": need[name],
                     "GB_per_s": round(need[name] / us / 1e3, 1)}
        print("%-10s %.2f us per launch, %.1f MB, %.0f GB/s" % (name, us, need[name] / 1e6, need[name] / us / 1e3),
              flush=True)
    assert eng.error_code() == 0
    eng.close()
    return out


def peak_memory(net, global_batch, n):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    try:
        eng = engine(net, "svd", {"svd_rank": 3}, n)
        x, y = batch(global_batch)
        eng.prepare(x, y, warmup=1)
        for _ in range(2):
            eng.train_step(x, y)
        torch.cuda.synchronize()
        err = eng.error_code()
        eng.close()
    except torch.cuda.OutOfMemoryError:
        return {"n": n, "micro_batch": global_batch // n, "peak_mib": None, "oom": True}
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    print("%s batch %d, N=%d: peak allocated %.0f MiB" % (net, global_batch, n, peak), flush=True)
    return {"n": n, "micro_batch": global_batch // n, "peak_mib": round(peak, 1), "error_code": err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/accumulate_h100_1gpu.json)")
    ap.add_argument("--micro", type=int, default=128)
    ap.add_argument("--ns", type=str, default="1,2,4,8")
    ap.add_argument("--time-steps", type=int, default=20)
    ap.add_argument("--time-reps", type=int, default=4)
    ap.add_argument("--kernel-reps", type=int, default=200)
    ap.add_argument("--mem-net", type=str, default="ResNet50")
    ap.add_argument("--mem-batch", type=int, default=1024)
    ap.add_argument("--mem-n", type=int, default=8)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    ns = [int(v) for v in a.ns.split(",")]
    rec = {"card": card(), "net": "ResNet18", "micro_batch": a.micro, "time_steps": a.time_steps, "timing": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for code, kw, label in CONFIGS:
        probe = engine("ResNet18", code, kw, 1, graph=False, code_stats=True)
        x, y = batch(a.micro)
        probe.prepare(x, y, warmup=0)
        probe.code_stats(reset=True)
        probe.train_step(x, y)
        push = probe.code_stats()["model"]["bytes"]
        probe.close()
        engs, data = {}, {}
        for n in ns:
            data[n] = batch(n * a.micro, seed=1)
            engs[n] = engine("ResNet18", code, kw, n)
            engs[n].prepare(*data[n], warmup=3)
        times = {n: [] for n in ns}
        for rep in range(a.time_reps + 1):
            for n in ns:
                torch.cuda.synchronize()
                ev0.record()
                for _ in range(a.time_steps):
                    engs[n].train_step(*data[n])
                ev1.record()
                torch.cuda.synchronize()
                if rep > 0:
                    times[n].append(ev0.elapsed_time(ev1) / a.time_steps)
        for n in ns:
            med = median(times[n])
            samples = n * a.micro
            row = {"code": label, "n": n, "samples_per_step": samples, "median_step_ms": round(med, 4),
                   "us_per_sample": round(1e3 * med / samples, 3), "step_ms": [round(v, 4) for v in times[n]],
                   "push_bytes_per_step": round(push), "push_bytes_per_sample": round(push / samples, 1),
                   "launches_per_step": engs[n].launches_per_step, "error_code": engs[n].error_code()}
            rec["timing"].append(row)
            print("%-16s N=%d  %.3f ms/step  %.3f us/sample  %.0f push B/sample  (%d launches)" % (
                label, n, med, row["us_per_sample"], row["push_bytes_per_sample"], row["launches_per_step"]),
                flush=True)
        for e in engs.values():
            e.close()
    rec["passes"] = time_passes(a.micro, a.kernel_reps)
    rec["memory"] = {"net": a.mem_net, "global_batch": a.mem_batch,
                     "points": [peak_memory(a.mem_net, a.mem_batch, n) for n in (1, a.mem_n)]}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
