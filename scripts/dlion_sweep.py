#!/usr/bin/env python
"""Distributed Lion against Signum and the PS-side Lion on the bf16 engine, one GPU.

* Step time (CUDA graph + overlap, batch ``--batch``) on ResNet-18 and VGG-11 of ``dlion`` with the vote and with the
  mean at betas (0.9, 0.99) and at b1 = 0, ``signum`` with beta 0.9, and ``--optimizer lion`` with the dense code, all
  engines of a net alternated in one process for ``--time-reps`` rounds after a warm-up round (every round's mean is
  kept, and the median).
* Push bytes per worker and step, from the plan: the sign bits (``signum_bytes``) and what travels dense
  (``dense_bytes``: bf16 weights of the dense code, fp32 vectors).
* The encode of every ResNet-18 backward group (``v2_dlion_encode`` at b1 = 0.9, next to ``v2_signum_encode`` at beta
  0.9), and the PS vote and mean kernels (``v2_ps_signum``) in a loopback arena of W = 1, 4, 8, 16 virtual workers, one
  owner and one group, timed with CUDA events over ``--ps-iters`` launches.

The card name and power limit are read in the same run.

    python scripts/dlion_sweep.py --out profiles/dlion_h100_1gpu.json
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
from signum_sweep import ps_vote_time  # noqa: E402

# (name, code, optimizer, engine keywords)
CONFS = [("dlion-vote", "dlion", "sgd", {"betas": (0.9, 0.99)}),
         ("dlion-mean", "dlion", "sgd", {"betas": (0.9, 0.99), "dlion_aggregate": "mean"}),
         ("dlion-vote-b1=0", "dlion", "sgd", {"betas": (0.0, 0.99)}),
         ("dlion-mean-b1=0", "dlion", "sgd", {"betas": (0.0, 0.99), "dlion_aggregate": "mean"}),
         ("signum", "signum", "sgd", {"momentum": 0.9}),
         ("lion-dense", "sgd", "lion", {})]


def engine(net, code, optimizer, kw):
    from atomo_b200.models import build_model
    from atomo_b200.runtime.shadow_engine import ShadowEngine
    torch.manual_seed(0)
    return ShadowEngine(build_model(net, 10), 0, 1, code=code, optimizer=optimizer, lr=1e-3, seed=1, **kw)


def encode_times(C, shapes, iters, n_groups=5):
    """Per backward group of ``shapes``: mean microseconds of one Signum (beta 0.9) and one Distributed Lion
    (b1 = 0.9) encode launch over the group's tiles and vector chunks, pushing into a local arena."""
    from atomo_b200.ops import plan2 as P
    dev = torch.device("cuda", 0)
    pl = P.build_plan2(shapes, "signum", n_owners=1, n_groups=n_groups)
    u8 = lambda b: torch.frombuffer(bytearray(b or b"\0" * 24), dtype=torch.uint8).to(dev)
    z = lambda n, dt=torch.float32: torch.zeros(n, dtype=dt, device=dev)
    t_units, t_enc = u8(pl.units_bytes()), u8(P.Plan2.tiles_bytes(pl.enc_tiles))
    chunks, vec_range = P.vec_chunks(pl)
    t_vchunks = u8(chunks)
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = [torch.randn(q.numel, device=dev, generator=g).to(torch.bfloat16) for q in pl.params if q.is_w]
    gptr = torch.tensor([t.data_ptr() for t in grads], dtype=torch.int64, device=dev)
    arena, sig = z(pl.arena_floats), z(1024, torch.int32)
    t_arena, t_sig = (torch.tensor([t.data_ptr()], dtype=torch.int64, device=dev) for t in (arena, sig))
    ctrl = u8(P.pack_ctrl2(step=1, lr=1e-3, seed=1))
    vgrads, mom, vmom = torch.randn(pl.v_total, device=dev, generator=g), z(pl.w_total), z(pl.v_total)
    counters = z(16, torch.int32)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for grp in range(pl.n_groups):
        (t0, nt), (v0, nv) = pl.enc_range[grp], vec_range[grp]
        common = (t_units.data_ptr(), t_enc.data_ptr(), t0, nt, gptr.data_ptr(), t_vchunks.data_ptr() + 24 * v0, nv,
                  vgrads.data_ptr(), mom.data_ptr(), vmom.data_ptr())
        tail = (t_arena.data_ptr(), t_sig.data_ptr(), 1, pl.arena_floats, 0, grp, ctrl.data_ptr(),
                counters.data_ptr() + 4 * grp, 0, grp == pl.n_groups - 1)
        launches = {"signum": lambda: C.v2_signum_encode(*common, 0.9, *tail),
                    "dlion": lambda: C.v2_dlion_encode(*common, 0.9, 0.99, *tail)}
        r = {"group": grp, "tiles": nt, "vector_chunks": nv,
             "weight_elements": sum(n for (_, _, n, _) in pl.enc_tiles[t0:t0 + nt])}
        for name, launch in launches.items():
            for _ in range(10):
                launch()
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(iters):
                launch()
            ev1.record()
            torch.cuda.synchronize()
            r[name + "_us"] = round(ev0.elapsed_time(ev1) * 1e3 / iters, 2)
        # bf16 gradient read, fp32 momentum read and written, 1 bit pushed per weight element
        r["bytes"] = 10 * r["weight_elements"] + r["weight_elements"] // 8
        r["dlion_GB_s"] = round(r["bytes"] / r["dlion_us"] / 1e3, 1)
        out.append(r)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="JSON record to write (profiles/dlion_h100_1gpu.json)")
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
           "timing": [], "push_bytes": [], "encode": [], "ps": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for net in a.nets.split(","):
        x, y = SyntheticImageDataset(input_shape(net), 10, 4096, seed=0).materialize(a.batch)
        x, y = x.pin_memory(), y.pin_memory()
        engs = {}
        for c in CONFS:
            engs[c[0]] = engine(net, *c[1:])
            engs[c[0]].prepare(x, y, warmup=3)
        times = {c[0]: [] for c in CONFS}
        for rep in range(a.time_reps + 1):
            for c in CONFS:
                torch.cuda.synchronize()
                ev0.record()
                for _ in range(a.time_steps):
                    engs[c[0]].train_step(x, y)
                ev1.record()
                torch.cuda.synchronize()
                if rep > 0:         # the first round warms every engine
                    times[c[0]].append(ev0.elapsed_time(ev1) / a.time_steps)
        for name, code, opt, kw in CONFS:
            v = sorted(times[name])
            e = engs[name]
            nbytes = e.plan.dense_bytes() + e.plan.signum_bytes()
            t = {"net": net, "config": name, "code": code, "optimizer": opt,
                 "settings": {k: list(v) if isinstance(v, tuple) else v for k, v in kw.items()},
                 "median_ms": round(v[len(v) // 2], 4), "step_ms": [round(s, 4) for s in times[name]],
                 "launches_per_step": e.launches_per_step, "error_code": e.error_code()}
            rec["timing"].append(t)
            rec["push_bytes"].append({"net": net, "config": name, "bytes": nbytes})
            print("%-8s %-16s step ms %.3f  push %.3f MB" % (net, name, t["median_ms"], nbytes / 2 ** 20), flush=True)
        for e in engs.values():
            e.close()
    C = load()
    shapes = [tuple(p.shape) for p in build_model("ResNet18", 10).parameters()]
    for r in encode_times(C, shapes, a.ps_iters):
        rec["encode"].append(r)
        print("encode group %d  signum %.1f us  dlion %.1f us  %.0f GB/s" % (r["group"], r["signum_us"], r["dlion_us"],
                                                                             r["dlion_GB_s"]), flush=True)
    for W in (1, 4, 8, 16):
        for mean in (False, True):
            r = ps_vote_time(C, shapes, W, a.ps_iters, mean=mean)
            r["aggregate"] = "mean" if mean else "vote"
            rec["ps"].append(r)
            print("ps %s W=%2d  %.1f us  %.0f GB/s" % (r["aggregate"], W, r["us"], r["GB_s"]), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
        f.write("\n")
    print("wrote", a.out, time.strftime("%Y-%m-%d %H:%M:%S"))


if __name__ == "__main__":
    main()
