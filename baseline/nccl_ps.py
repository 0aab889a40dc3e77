"""The comparator: the reference ALGORITHM re-hosted on torch.distributed/NCCL.

The reference itself cannot run here (Python-2.7 + mpi4py + torch-0.3, not
pip-installable, default coder module missing — DESIGN.md), so BASELINE.md names
this as the bar: the same synchronous-PS protocol and the same per-tensor
spectral-ATOMO coder, with MPI replaced by NCCL and LAPACK by
``torch.linalg.svd`` (cuSOLVER) on the GPU — i.e. what a straightforward port of
``sync_replicas_master_nn.py`` / ``distributed_worker.py`` gives on an H100 box:

  rank 0 = dedicated PS (like the reference), ranks 1..N-1 = workers;
  per step: ``dist.broadcast`` of the flat fp32 parameters -> eager fp32
  forward/backward -> per-tensor ``SVD.encode`` (torch.linalg.svd + host-side
  Bernoulli sampling, svd.py:79-118) -> one packed NCCL send per worker -> PS
  decodes ``(u*s)@vT`` per (layer, worker), averages, ``optim.SGD.step``.

With one GPU the PS and the single worker share the device (no communication).
None of the sm_90a kernels, the symmetric heap or CUDA graphs are used here.
"""
from __future__ import annotations

import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_baseline(args, rank, world, dev):
    from atomo_b200 import codings
    from atomo_b200.data import SyntheticImageDataset
    from atomo_b200.models import build_model, input_shape
    from atomo_b200.optim import SGD
    from atomo_b200.parallel import wire
    from atomo_b200.runtime.flat import FlatLayout, bind_parameters

    torch.manual_seed(0)
    torch.backends.cudnn.benchmark = True
    model = build_model(args.network, 10, "Cifar10").to(dev)
    bf16 = getattr(args, "dtype", "fp32") == "bf16"     # same model-compute precision as the product arm when asked
    layout = FlatLayout.from_module(model)
    flat = torch.zeros(layout.total, device=dev)
    bind_parameters(model, flat, layout)
    if bf16:
        model = model.to(memory_format=torch.channels_last)
        bind_parameters(model, flat, layout)
    is_ps = rank == 0
    is_worker = world == 1 or rank > 0
    nworkers = max(world - 1, 1)
    code = args.code if args.code != "sgd" else "sgd"
    # gram_route=False: the comparator stays what BASELINE.md names, torch.linalg.svd per tensor
    enc = codings.build(code, rank=args.svd_rank, random_sample=True, gram_route=False) if code == "svd" else codings.build(code)
    dec = codings.build(code, rank=args.svd_rank, random_sample=False, gram_route=False) if code == "svd" else codings.build(code)
    opt = SGD(model.parameters(), lr=args.lr, momentum=args.momentum) if is_ps else None
    shape = input_shape(args.network, "Cifar10")
    xs, ys = SyntheticImageDataset(shape, 10, 50000, seed=rank).materialize(args.batch_size)
    host_x, host_y = xs.pin_memory(), ys.pin_memory()
    crit = torch.nn.CrossEntropyLoss()
    shapes = [tuple(p.shape) for p in model.parameters()]
    loss_val = 0.0

    def one_step(from_host: bool):
        nonlocal loss_val
        if world > 1:
            dist.broadcast(flat, src=0)
        codes = None
        if is_worker:
            x = host_x.to(dev, non_blocking=True) if from_host else xd
            y = host_y.to(dev, non_blocking=True) if from_host else yd
            model.zero_grad(set_to_none=True)
            if bf16:
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    loss = crit(model(x.contiguous(memory_format=torch.channels_last)).float(), y)
            else:
                loss = crit(model(x), y)
            loss.backward()
            codes = [enc.encode(p.grad) for p in model.parameters()]
            if from_host:
                loss_val = float(loss.item())  # D2H read of the step's result
            if world > 1:
                buf = wire.pack({"codes": codes}, device=dev)
                dist.send(torch.tensor([buf.numel()], dtype=torch.int64, device=dev), dst=0)
                dist.send(buf, dst=0)
        if is_ps:
            agg = [torch.zeros(s, device=dev) for s in shapes]
            if world == 1:
                msgs = [codes]
            else:
                msgs = []
                for w in range(1, world):
                    n = torch.zeros(1, dtype=torch.int64, device=dev)
                    dist.recv(n, src=w)
                    buf = torch.empty(int(n.item()), dtype=torch.uint8, device=dev)
                    dist.recv(buf, src=w)
                    msgs.append(wire.unpack(buf)["codes"])
            for m in msgs:
                for i, c in enumerate(m):
                    agg[i] += dec.decode(c).reshape(shapes[i])
            opt.step(grads=[g / len(msgs) for g in agg], cuda=True)

    xd, yd = host_x.to(dev), host_y.to(dev)

    def barrier():
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    def timed(nsteps, from_host):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(nsteps):
            one_step(from_host)
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1)
        if world > 1:
            t = torch.tensor([ms], dtype=torch.float64, device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms

    for _ in range(max(args.warmup, 3)):
        one_step(False)
    ms = timed(args.steps, False)
    ms_e2e = timed(args.steps, True)
    imgs = nworkers * args.batch_size
    if rank == 0:
        print(json.dumps({
            "metric": "ResNet-18 CIFAR-10 images/sec (whole box, device-timed, max over ranks)",
            "value": round(imgs * args.steps / (ms / 1e3), 2), "unit": "images/s", "n_gpus": world,
            "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": round(ms / args.steps, 3),
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16" if bf16 else "fp32",
            "data": "synthetic",
            "impl": "nccl-baseline",
            "config": {"model": args.network, "global_batch": imgs, "per_worker_batch": args.batch_size,
                       "parallelism": "dedicated ps + %d workers" % nworkers if world > 1 else "ps+worker on one gpu",
                       "code": code, "svd_rank": args.svd_rank,
                       "stack": "torch.distributed NCCL send/recv/broadcast + torch.linalg.svd + eager %s" %
                                ("bf16 autocast, NHWC" if bf16 else "fp32")},
            "e2e": {"value": round(imgs * args.steps / (ms_e2e / 1e3), 2), "unit": "images/s",
                    "ms_per_step": round(ms_e2e / args.steps, 3),
                    "h2d_bytes_per_step": host_x.numel() * 4 + host_y.numel() * 8, "d2h_bytes_per_step": 4},
            "gpu_launches": 0}))
    if world > 1:
        dist.destroy_process_group()
