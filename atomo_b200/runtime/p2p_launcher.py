"""``--backend p2p``: the launcher side of the fused NVLink engines.

Counterpart of the role dispatch in ``/root/reference/src/distributed_nn.py:243-260`` plus the training loops of
``sync_replicas_master_nn.py:173-234`` / ``distributed_worker.py:166-262``: data sharding, LR shrinkage every
``--shrinkage-freq`` steps (applied to the optimizer — the reference only printed it), periodic evaluation,
checkpoints in the ``model_step_<N>`` layout, and the reference's log lines with REAL per-phase numbers taken from
device-side timers (``Comp`` / ``Encode`` / ``Comm`` on the worker line, ``Decode Cost`` / ``Gather`` on the PS line).

Engine choice (``--engine auto``): ``--dtype bf16`` with ``--code svd|qsvd|sgd|topk|sign|powersgd|fp8`` runs the
overlapped, sharded
``ShadowEngine``; everything else (fp32, qsgd / terngrad / entrywise) runs the fp32-flat ``FusedEngine``.
``--engine shadow`` also runs ``--code qsgd|terngrad`` on ``ShadowEngine`` (bf16 only) and refuses ``--code
entrywise``, which the launcher keeps on ``FusedEngine``; ``--engine fused`` always picks ``FusedEngine``.  ``--code
topk``, ``--code sign``, ``--code powersgd`` and ``--code fp8`` exist only on ``ShadowEngine``.
"""
from __future__ import annotations

import os
import time

import torch
import torch.distributed as dist
import torch.nn.functional as F


class _HostEvent:
    """perf_counter stand-in for torch.cuda.Event when the loop runs on a CPU stand-in engine (tests)."""

    def record(self):
        self.t = time.perf_counter()

    def elapsed_time(self, other) -> float:
        return (other.t - self.t) * 1e3


def _build_engine(args, model, rank, world):
    engine = getattr(args, "engine", "auto")
    code = args.code.lower()
    if code == "topk" and (engine == "fused" or args.dtype != "bf16"):
        raise SystemExit("--code topk runs on the bf16 engine only (--dtype bf16, --engine auto|shadow); the fp32-flat "
                         "engine has no top-k selection")
    if code == "sign" and (engine == "fused" or args.dtype != "bf16"):
        raise SystemExit("--code sign runs on the bf16 engine only (--dtype bf16, --engine auto|shadow); the fp32-flat "
                         "engine has no scaled-sign code")
    if code == "fp8" and (engine == "fused" or args.dtype != "bf16"):
        raise SystemExit("--code fp8 runs on the bf16 engine only (--dtype bf16, --engine auto|shadow); the fp32-flat "
                         "engine has no fp8 code")
    if code == "powersgd" and (engine == "fused" or args.dtype != "bf16"):
        raise SystemExit("--code powersgd runs on the bf16 engine only (--dtype bf16, --engine auto|shadow); the "
                         "fp32-flat engine has no PowerSGD code")
    if code == "powersgd" and not 1 <= args.svd_rank <= 4:
        raise SystemExit("--code powersgd needs --svd-rank in [1, 4] (the rank of the pushed factors; got %d)"
                         % args.svd_rank)
    if engine == "auto":
        shadow = args.dtype == "bf16" and code in ("svd", "qsvd", "sgd", "dense", "lossless", "topk", "sign",
                                                   "powersgd", "fp8")
    elif engine == "shadow":
        if args.dtype != "bf16":
            raise SystemExit("--engine shadow trains bf16 weights: it needs --dtype bf16 (fp32 runs on --engine fused)")
        if code not in ("svd", "qsvd", "sgd", "dense", "lossless", "qsgd", "terngrad", "topk", "sign", "powersgd",
                        "fp8"):
            raise SystemExit("--engine shadow runs --code svd|qsvd|sgd|qsgd|terngrad|topk|sign|powersgd|fp8; --code %s "
                             "runs on --engine fused" % args.code)
        shadow = True
    else:
        shadow = False
    if shadow:
        from .shadow_engine import ShadowEngine
        kw = {}
        if code in ("qsgd", "terngrad"):
            kw = dict(quantization_level=args.quantization_level, bucket_size=args.bucket_size)
        elif code == "topk":
            kw = dict(entry_budget=args.entry_budget)
        elif code in ("sign", "fp8"):
            kw = dict(bucket_size=args.bucket_size)
        if getattr(args, "code_stats", False):
            if code == "qsvd":
                raise SystemExit("--code-stats does not model QSVD's int8 left factors (use --code svd)")
            kw["code_stats"] = True
        if getattr(args, "error_feedback", False):
            kw["error_feedback"] = True      # the engine refuses codes / --num-aggregate it cannot feed back
        return ShadowEngine(model, rank, world, code=args.code, svd_rank=args.svd_rank, lr=args.lr,
                            momentum=args.momentum, weight_decay=args.weight_decay, nesterov=args.nesterov,
                            optimizer=args.optimizer, ps_mode=args.ps_mode, groups=args.groups, sampling=args.sampling,
                            prob_rule=args.prob_rule, seed=args.seed, num_aggregate=args.num_aggregate,
                            timeout_s=args.flag_timeout, **kw), "shadow"
    from .engine import FusedEngine
    if getattr(args, "error_feedback", False):
        raise SystemExit("--error-feedback runs on the bf16 engine (--dtype bf16, --engine auto|shadow); the fp32-flat "
                         "engine keeps no residual (run without --error-feedback)")
    if getattr(args, "code_stats", False):
        raise SystemExit("--code-stats reads the statistics of the bf16 engine (--dtype bf16, --engine auto|shadow); "
                         "the fp32-flat engine does not compute them (run without --code-stats)")
    if args.optimizer != "sgd":
        raise SystemExit("--optimizer adam on the p2p backend needs --dtype bf16 with --code svd|sgd, or --engine "
                         "shadow with --code qsgd|terngrad (ShadowEngine); the fp32-flat engine fuses momentum-SGD only")
    ps_mode = "colocated" if args.ps_mode == "sharded" else args.ps_mode
    return FusedEngine(model, rank, world, code=args.code, svd_rank=args.svd_rank, lr=args.lr, momentum=args.momentum,
                       weight_decay=args.weight_decay, nesterov=args.nesterov, ps_mode=ps_mode,
                       sampling=args.sampling, prob_rule=args.prob_rule, seed=args.seed,
                       quantization_level=args.quantization_level, bucket_size=args.bucket_size,
                       entry_budget=args.entry_budget, dtype=args.dtype, channels_last=(args.dtype == "bf16"),
                       timeout_s=args.flag_timeout), "fused"


def run_p2p_training(args, device=None):
    """``device`` is for the CPU tests of this loop (a stand-in engine on ``cpu``); real runs leave it None."""
    from ..data import DataLoader, build_datasets, shard_dataset
    from ..models import build_model
    from ..utils import checkpoint as ckpt
    from ..utils.logging import MetricsWriter, master_line, test_line, worker_line
    from .nn_ops import accuracy

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", str(rank)))
    dev = torch.device(device) if device is not None else torch.device("cuda", local_rank)
    on_gpu = dev.type == "cuda"
    if on_gpu:
        torch.cuda.set_device(local_rank)
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", args.master_addr)
        os.environ.setdefault("MASTER_PORT", str(args.master_port))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    torch.manual_seed(args.seed)
    train_set, test_set, num_classes = build_datasets(
        args.dataset, args.data_root, synthetic=args.synthetic, seed=args.seed,
        train_len=args.train_len or None, test_len=args.test_len or None)
    model = build_model(args.network, num_classes, args.dataset)
    eng, kind = _build_engine(args, model, rank, world)
    metrics = MetricsWriter(getattr(args, "metrics_file", ""), rank, "p2p")
    first = eng.first_worker
    nworkers = eng.W
    shard = shard_dataset(train_set, max(rank - first, 0), nworkers, seed=args.seed)
    if getattr(args, "gpu_data", False):
        from ..data.gpu_loader import GpuLoader
        # the layout each engine's static input has: channels_last on the shadow engine, as the CPU batches otherwise
        loader = GpuLoader(shard, args.batch_size, args.dataset, train=True, seed=args.seed + rank, device=dev,
                           channels_last=kind == "shadow")
        test_loader = GpuLoader(test_set, args.test_batch_size, args.dataset, train=False, device=dev,
                                channels_last=kind == "shadow")
    else:
        loader = DataLoader(shard, batch_size=args.batch_size, shuffle=True, seed=args.seed + rank, drop_last=True,
                            pin_memory=True, prefetch=2)
        test_loader = torch.utils.data.DataLoader(test_set, batch_size=args.test_batch_size, shuffle=False)
    x0, y0 = loader.next_batch()
    eng.prepare(x0, y0, warmup=2 if args.max_steps < 8 else 3)   # eager warm-up steps (cuDNN autotune) count as steps
    if getattr(args, "resume", False):
        last = ckpt.latest_step(args.train_dir)
        if last is not None:
            eng.load_checkpoint(args.train_dir, last)   # collective: same directory on every rank
    n_data, base_lr = len(shard), args.lr
    freq = max(int(args.shrinkage_freq), 1)
    # LR schedule derived from the step (also right after --resume): base * shrinkage ** (completed steps // freq)
    eng.set_lr(base_lr * args.lr_shrinkage ** ((eng.step - 1) // freq))
    if kind == "shadow":
        msg_mb = (eng.plan.expected_factor_bytes() + eng.plan.dense_bytes()) / 2 ** 20
    else:
        msg_mb = (eng.plan.factor_bytes_per_worker() + eng.plan.dense_bytes()) / 2 ** 20
    ev_a, ev_b = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) if on_gpu else \
        (_HostEvent(), _HostEvent())
    ev_a.record()
    since = 0
    eng.phase_stats(reset=True)
    if getattr(args, "code_stats", False) and eng.is_worker:
        eng.code_stats(reset=True)              # the first record covers the logged steps only, like phase_stats

    def collective_barrier():
        if on_gpu:
            torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()

    while eng.step <= args.max_steps:
        x, y = loader.next_batch()
        stats = eng.train_step(x, y)
        cur = eng.step - 1
        since += 1
        if cur % args.log_interval == 0 or cur == args.max_steps:
            ev_b.record()
            loss, p1, p5 = stats.tolist()            # D2H sync: everything up to `cur` has finished
            step_s = ev_a.elapsed_time(ev_b) / max(since, 1) / 1e3
            ph = eng.phase_stats(reset=True)
            err = eng.error_code()                   # sticky device-side error (spin-wait timeout, stale slot, NaN)
            if err:
                raise SystemExit("rank %d: device-side error code %d at step %d: aborting (parameters can no longer "
                                 "be trusted; resume from the last checkpoint)" % (rank, err, cur))
            enc = ph.get("encode_us", 0.0) / 1e6
            comm = (ph.get("param_wait_us", 0.0) + max(ph.get("to_params_us", 0.0) - ph.get("to_push_us", 0.0), 0.0)) / 1e6
            comp = max(step_s - comm, 0.0) if kind == "fused" else max(ph.get("to_push_us", 0.0) / 1e6, 0.0)
            if eng.is_worker:
                print(worker_line(rank, cur, loader.epochs_completed, (cur * args.batch_size) % n_data, n_data, loss,
                                  step_s, comp, enc, comm, msg_mb, p1, p5))
            if eng.is_ps or (kind == "shadow" and eng.is_owner):
                print(master_line(cur, ph.get("ps_work_us", 0.0) / 1e6, eng.lr, ph.get("ps_wait_push_us", 0.0) / 1e6))
            extra = {}
            if getattr(args, "code_stats", False) and eng.is_worker:
                extra["code_stats"] = eng.code_stats(reset=True)
            if getattr(args, "error_feedback", False) and eng.is_worker:
                extra["ef_norm"] = eng.error_feedback_norm()["model"]
            metrics.write(step=cur, loss=loss, prec1=p1, prec5=p5, step_s=step_s, comp=comp, encode=enc, comm=comm,
                          msg_mb=msg_mb, lr=eng.lr, phase_us={k: round(float(v), 1) for k, v in ph.items()}, **extra)
            ev_a.record()
            since = 0
        if cur % args.eval_freq == 0:
            # every rank enters: nobody is left spinning on a device flag while one rank evaluates / writes files
            collective_barrier()
            # every rank calls it: a rank that TRAINS writes the evaluator's file (real BN running statistics; the
            # reference's PS checkpoints carry untrained ones, SURVEY 2.9), the PS side writes the optimizer sidecar
            eng.save_checkpoint(args.train_dir, cur)
            if eng.is_worker and rank == first:
                eng.model.eval()
                tl, a1, a5, nbt, cnt = 0.0, 0.0, 0.0, 0, 0
                with torch.no_grad():
                    for i, (dx, dy) in enumerate(test_loader):
                        if args.eval_batches and i >= args.eval_batches:
                            break
                        dx, dy = dx.to(dev), dy.to(dev)
                        if kind == "shadow":
                            dx = dx.contiguous(memory_format=torch.channels_last)
                            with torch.autocast("cuda", dtype=torch.bfloat16):
                                out = eng.model(dx).float()
                        else:
                            out = eng.model(dx)
                        tl += F.cross_entropy(out, dy, reduction="sum").item()
                        b1, b5 = accuracy(out, dy, (1, 5))
                        a1 += b1.item(); a5 += b5.item(); nbt += 1; cnt += len(dy)
                print(test_line(cur, tl / max(cnt, 1), a1 / max(nbt, 1), a5 / max(nbt, 1)))
                eng.model.train()
            collective_barrier()
        if (eng.step - 1) % freq == 0:          # shrinkage (master:232-234), actually applied to the optimizer
            eng.set_lr(base_lr * args.lr_shrinkage ** ((eng.step - 1) // freq))
    err = eng.error_code()
    if err:
        print("rank %d: device error code %d" % (rank, err))
    loader.close()
    metrics.close()
    eng.close()
    if world > 1:
        dist.destroy_process_group()
