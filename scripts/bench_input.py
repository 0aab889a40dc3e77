#!/usr/bin/env python
"""Training throughput of the p2p launcher's input paths on one GPU: ResNet-18, batch 128, the shadow engine
(spectral ATOMO, rank 3, as in bench.py's headline).

  (a) cpu:      data.loader.DataLoader as run_p2p_training builds it (PIL transforms, pinned staging) -> train_step
  (b) gpu:      data.gpu_loader.GpuLoader (--gpu-data)                                           -> train_step
  (c) resident: train_step() on inputs already in the engine's static buffer (bench.py's upper bound)

each over a CIFAR-10-format UInt8ImageDataset with the real CIFAR-10 training transform and over the synthetic
CIFAR-10 set.  Also times the augment_gather kernel alone with CUDA events (bytes: B*C*H*W in for uint8, 4x that
for fp32; 4*B*C*H*W + 8*B out) and records the card name and power limit read in the same run.

    python scripts/bench_input.py [--steps 200] [--cpu-steps 40] [--kernel-iters 2000] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from atomo_b200.data import DataLoader, GpuLoader, SyntheticImageDataset, UInt8ImageDataset, real_transforms  # noqa
from atomo_b200.models import build_model  # noqa: E402
from atomo_b200.runtime.shadow_engine import ShadowEngine  # noqa: E402

BATCH = 128


def card(dev):
    q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(dev)


def images_per_s(eng, feed, steps, warmup, dev):
    for _ in range(warmup):
        eng.train_step(*feed())
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for _ in range(steps):
        eng.train_step(*feed())
    torch.cuda.synchronize(dev)
    return BATCH * steps / (time.perf_counter() - t0)


def kernel_time(gl, iters, dev):
    """Mean time of one augment_gather launch building a batch of BATCH, and its bytes moved."""
    _, h, w, c = gl.src.shape
    x = torch.empty((BATCH, c, h, w), device=dev, memory_format=torch.channels_last)
    y = torch.empty(BATCH, dtype=torch.int64, device=dev)
    s = gl.spec

    def launch(i):
        pos = (i * BATCH) % (len(gl) * BATCH)
        gl._C.augment_gather(gl.src, gl.labels, gl._order, pos, gl.mean_std, s.pad, s.reflect, s.augment, gl.seed, 0,
                             None, x, y)
    for i in range(50):
        launch(i)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        launch(i)
    e1.record()
    torch.cuda.synchronize(dev)
    us = e0.elapsed_time(e1) * 1e3 / iters
    elems = BATCH * c * h * w
    nbytes = elems * gl.src.element_size() + 4 * elems + 8 * BATCH
    return {"us_per_batch": round(us, 3), "bytes": nbytes, "GB_per_s": round(nbytes / us / 1e3, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed steps of (b) and (c)")
    ap.add_argument("--cpu-steps", type=int, default=40, help="timed steps of (a)")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--kernel-iters", type=int, default=2000)
    ap.add_argument("--train-len", type=int, default=50000)
    ap.add_argument("--out", type=str, default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_input.py measures on a CUDA GPU; none is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(dev), "network": "ResNet18", "batch": BATCH, "engine": "shadow", "code": "svd", "rank": 3,
           "cpu_threads": torch.get_num_threads()}

    rng = np.random.default_rng(0)
    n = args.train_len
    sets = {
        "cifar10_uint8": UInt8ImageDataset(rng.integers(0, 256, size=(n, 32, 32, 3), dtype=np.uint8),
                                           (np.arange(n) % 10).tolist(), real_transforms("cifar10")[0]),
        "synthetic": SyntheticImageDataset((3, 32, 32), 10, n, seed=0),
    }
    torch.manual_seed(0)
    eng = ShadowEngine(build_model("ResNet18", 10), 0, 1, code="svd", svd_rank=3, lr=0.01, momentum=0.9)
    x0, y0 = SyntheticImageDataset((3, 32, 32), 10, 256).materialize(BATCH)
    eng.prepare(x0.pin_memory(), y0.pin_memory(), warmup=3)

    for name, ds in sets.items():
        r = {}
        cpu = DataLoader(ds, batch_size=BATCH, shuffle=True, seed=1, drop_last=True, pin_memory=True, prefetch=2)
        r["a_cpu_loader"] = round(images_per_s(eng, cpu.next_batch, args.cpu_steps, args.warmup, dev), 1)
        cpu.close()
        t0 = time.perf_counter()
        gl = GpuLoader(ds, BATCH, "cifar10", train=True, seed=1, device=dev, channels_last=True)
        r["gpu_loader_upload_s"] = round(time.perf_counter() - t0, 2)
        for rep in range(3):           # (b) and (c) alternate: other work shares the host
            r.setdefault("b_gpu_loader", []).append(
                round(images_per_s(eng, gl.next_batch, args.steps, args.warmup, dev), 1))
            r.setdefault("c_resident", []).append(round(images_per_s(eng, tuple, args.steps, args.warmup, dev), 1))
        r["kernel"] = kernel_time(gl, args.kernel_iters, dev)
        gl.close()
        res[name] = r
        print(name, json.dumps(r), flush=True)
    err = eng.error_code()
    eng.close()
    if err:
        raise SystemExit("device-side error code %d" % err)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
