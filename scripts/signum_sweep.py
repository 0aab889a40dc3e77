#!/usr/bin/env python
"""Signum with majority vote against the dense code and scaled sign on the bf16 engine, one GPU.

* Step time (CUDA graph + overlap, batch ``--batch``) on ResNet-18 and VGG-11 of the dense code (``sgd``), ``sign``
  (bucket 512) with error feedback off and on, and ``signum`` with beta 0 and 0.9, all engines of a net alternated in
  one process for ``--time-reps`` rounds after a warm-up round (every round's mean is kept, and the median).
* Push bytes per worker and step, from the plan: the sign bits (``signum_bytes``), the words and scales of sign
  (``qsgd_bytes``) and what travels dense (``dense_bytes``: bf16 weights of the dense code, fp32 vectors).
* The PS vote kernel alone (``v2_ps_signum``) in a loopback arena of W = 1, 4, 8, 16 virtual workers holding random
  bits of every ResNet-18 weight, one owner and one group, timed with CUDA events over ``--ps-iters`` launches.

The card name and power limit are read in the same run.

    python scripts/signum_sweep.py --out profiles/signum_h100_1gpu.json
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

CONFS = [("sgd", False, 0.9), ("sign", False, 0.9), ("sign", True, 0.9), ("signum", False, 0.0),
         ("signum", False, 0.9)]


def engine(net, code, ef, beta):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    lr = 1e-3 if code == "signum" else 0.05
    kw = {"bucket_size": 512} if code == "sign" else {}
    return ShadowEngine(build_model(net, 10), 0, 1, code=code, lr=lr, momentum=beta, seed=1, error_feedback=ef, **kw)


def push_bytes(pl):
    return pl.dense_bytes() + pl.qsgd_bytes() + pl.signum_bytes()


def ps_vote_time(C, shapes, W, iters, mean=False):
    """Mean microseconds of one v2_ps_signum launch over every tile of ``shapes`` (one group, one owner); ``mean``
    times the mean kernel of Distributed Lion instead of the vote."""
    from atomo_b200.ops import plan2 as P
    dev = torch.device("cuda", 0)
    pl = P.build_plan2(shapes, "signum", n_owners=1, n_groups=1)
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
    z = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device=dev)
    t_units, t_ps = u8(pl.units_bytes()), u8(P.Plan2.tiles_bytes(pl.ps_tiles))
    g = torch.Generator(device="cuda").manual_seed(W)
    arena = torch.randint(-2 ** 31, 2 ** 31 - 1, (pl.arena_floats * W,), dtype=torch.int32, device=dev,
                          generator=g).view(torch.float32)
    for w in range(W):            # fresh stamps, finite status words
        for u in pl.units:
            if u.kind == P.KIND_SIGNUM:
                base = w * pl.arena_floats + u.slot_off
                arena[base:base + u.n_ps].view(torch.int32).fill_(1)
                so = base + P.qsgd_norms_off(u.n_ps)
                arena[so:so + u.rows].zero_()
    sig = z(1024, torch.int32)
    sig[:W] = 1                   # push flags of group 0 for step 1
    ctrl = u8(P.pack_ctrl2(step=1, lr=1e-3, seed=1))
    master = torch.randn(pl.w_total, device=dev, generator=g)
    mom, vmom = z(pl.w_total), z(pl.v_total)
    wshadow = master.to(torch.bfloat16)
    vparams = torch.randn(pl.v_total, device=dev, generator=g)
    vgrads = [torch.randn(pl.v_total, device=dev, generator=g) for _ in range(W)]
    i64 = lambda xs: torch.tensor(list(xs), dtype=torch.int64, device=dev)
    t_wsh, t_vp, t_vg = i64([wshadow.data_ptr()]), i64([vparams.data_ptr()]), i64(t.data_ptr() for t in vgrads)
    t_sig = i64([sig.data_ptr()])
    counter = z(4, torch.int32)
    t0, nt = pl.ps_range[0][0]
    sm = torch.cuda.get_device_properties(dev).multi_processor_count

    def launch():
        C.v2_ps_signum(t_units.data_ptr(), t_ps.data_ptr(), t0, nt, W, 1, 0, True, 0, master.data_ptr(),
                       mom.data_ptr(), 0, 0, vmom.data_ptr(), 0, 0, 0, t_wsh.data_ptr(), vparams.data_ptr(), 0,
                       t_vp.data_ptr(), 0, t_vg.data_ptr(), arena.data_ptr(), pl.arena_floats, sig.data_ptr(),
                       t_sig.data_ptr(), ctrl.data_ptr(), counter.data_ptr(), int(5e9), 0, 1.0 / W,
                       max(1, min(3 * sm, nt)), mean=mean)
    for _ in range(10):
        launch()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(iters):
        launch()
    ev1.record()
    torch.cuda.synchronize()
    assert int(ctrl.view(torch.int32)[1]) == 0
    us = ev0.elapsed_time(ev1) * 1e3 / iters
    n_w = sum(u.numel for u in pl.units if u.kind == P.KIND_SIGNUM)
    # bits of W workers read; master and PS momentum read and written; the bf16 copy written
    nbytes = W * pl.signum_bytes() + 16 * n_w + 2 * n_w
    return {"W": W, "us": round(us, 2), "weight_elements": n_w, "bytes": nbytes, "GB_s": round(nbytes / us / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/signum_h100_1gpu.json)")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--time-steps", type=int, default=100)
    ap.add_argument("--time-reps", type=int, default=5)
    ap.add_argument("--ps-iters", type=int, default=200)
    ap.add_argument("--nets", type=str, default="ResNet18,VGG11")
    a = ap.parse_args()
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.ops._ext import load
    torch.cuda.set_device(0)
    rec = {"card": card(), "batch": a.batch, "time_steps": a.time_steps, "time_reps": a.time_reps,
           "timing": [], "push_bytes": [], "ps_vote": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for net in a.nets.split(","):
        x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(a.batch)
        x, y = x.pin_memory(), y.pin_memory()
        engs = {}
        for c in CONFS:
            engs[c] = engine(net, *c)
            engs[c].prepare(x, y, warmup=3)
        times = {c: [] for c in CONFS}
        for rep in range(a.time_reps + 1):
            for c in CONFS:
                torch.cuda.synchronize()
                ev0.record()
                for _ in range(a.time_steps):
                    engs[c].train_step(x, y)
                ev1.record()
                torch.cuda.synchronize()
                if rep > 0:         # the first round warms every engine
                    times[c].append(ev0.elapsed_time(ev1) / a.time_steps)
        for c in CONFS:
            v = sorted(times[c])
            e = engs[c]
            t = {"net": net, "code": c[0], "error_feedback": c[1], "momentum": c[2],
                 "median_ms": round(v[len(v) // 2], 4), "step_ms": [round(s, 4) for s in times[c]],
                 "launches_per_step": e.launches_per_step, "error_code": e.error_code()}
            rec["timing"].append(t)
            rec["push_bytes"].append({"net": net, "code": c[0], "bytes": push_bytes(e.plan)})
            print("%-8s %-6s ef=%d beta=%.1f  step ms %.3f  push %.3f MB" % (
                net, c[0], c[1], c[2], t["median_ms"], push_bytes(e.plan) / 2 ** 20), flush=True)
        for e in engs.values():
            e.close()
    C = load()
    shapes = [tuple(p.shape) for p in build_model("ResNet18", 10).parameters()]
    for W in (1, 4, 8, 16):
        r = ps_vote_time(C, shapes, W, a.ps_iters)
        rec["ps_vote"].append(r)
        print("ps vote W=%2d  %.1f us  %.0f GB/s" % (W, r["us"], r["GB_s"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
