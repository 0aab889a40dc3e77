"""Job launcher (parity: ``/root/reference/src/distributed_nn.py``).

``python -m atomo_b200.distributed_nn --network ResNet18 --dataset Cifar10
--code svd --svd-rank 3 ...`` with the reference's flags.  Instead of
``mpirun -n N --hostfile``, ranks come from ``torchrun`` (env RANK/WORLD_SIZE)
or from ``--nproc N`` (self-spawn on this host).  Role dispatch is the
reference's: rank 0 -> ``SyncReplicasMaster_NN``, rank>0 -> ``DistributedWorker``
(launcher:243-260) for the gloo/nccl backends; ``--backend p2p`` runs the fused
NVLink engine where every GPU trains and GPU 0 also hosts the PS.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch
import torch.distributed as dist

from .data import DataLoader, build_datasets, shard_dataset
from .parallel.transport import TorchDistTransport
from .runtime import DistributedWorker, SyncReplicasMaster_NN
from .utils.flags import add_fit_args


def _kwargs(args, role: str) -> dict:
    kw = {
        "batch_size": args.batch_size, "learning_rate": args.lr, "max_epochs": args.epochs,
        "max_steps": args.max_steps, "momentum": args.momentum, "network": args.network,
        "dataset": args.dataset, "comm_method": args.comm_type, "eval_freq": args.eval_freq,
        "train_dir": args.train_dir, "compress": args.compress, "enable_gpu": args.enable_gpu and not args.no_cuda,
        "code": args.code, "svd_rank": args.svd_rank, "quantization_level": args.quantization_level,
        "bucket_size": args.bucket_size, "entry_budget": args.entry_budget, "sampling": args.sampling,
        "prob_rule": args.prob_rule, "eval_batches": args.eval_batches or None,
        "metrics_file": args.metrics_file,
    }
    if role == "master":
        kw.update({"num_aggregate": args.num_aggregate, "lr_shrinkage": args.lr_shrinkage,
                   "optimizer": args.optimizer, "weight_decay": args.weight_decay, "nesterov": args.nesterov,
                   "trust_coefficient": getattr(args, "trust_coefficient", 0.001),
                   "lion_betas": tuple(getattr(args, "lion_betas", (0.9, 0.99))),
                   "clip_grad_norm": getattr(args, "clip_grad_norm", 0.0),
                   "ema_decay": getattr(args, "ema_decay", 0.0),
                   "resume": args.resume, "kill_stragglers": args.straggler_kill})
    else:
        kw["split_backward"] = args.straggler_kill
    return kw


def run_rank(args) -> None:
    if os.environ.get("ATOMO_HANG_DUMP_S"):  # hang diagnostics: dump all thread stacks after N s
        import faulthandler
        faulthandler.dump_traceback_later(float(os.environ["ATOMO_HANG_DUMP_S"]), exit=True)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", str(rank)))
    use_gpu = args.enable_gpu and not args.no_cuda and torch.cuda.is_available()
    backend = args.backend
    if backend == "auto":
        backend = "nccl" if use_gpu else "gloo"
    if use_gpu:
        torch.cuda.set_device(local_rank % torch.cuda.device_count())
    torch.manual_seed(args.seed + rank)

    if backend == "p2p":
        from .runtime.engine import run_p2p_training
        return run_p2p_training(args)
    if getattr(args, "gpu_data", False):
        raise SystemExit("--gpu-data builds batches for the --backend p2p engines; the %s backend's workers read "
                         "the CPU loader (run without --gpu-data)" % backend)
    if getattr(args, "error_feedback", False):
        raise SystemExit("--error-feedback keeps its residuals in the --backend p2p bf16 engine; the %s backend's "
                         "PyTorch coders do not (run without --error-feedback)" % backend)
    if getattr(args, "momentum_correction", False):
        raise SystemExit("--momentum-correction keeps each worker's momentum in the --backend p2p bf16 engine; the %s "
                         "backend's workers keep none (run without --momentum-correction)" % backend)
    if getattr(args, "accumulate_steps", 1) != 1:
        raise SystemExit("--accumulate-steps runs on the --backend p2p bf16 engine; the %s backend's workers push "
                         "after every backward (run without --accumulate-steps)" % backend)
    if args.code.lower() == "fp8":
        raise SystemExit("--code fp8 runs on the --backend p2p bf16 engine (--dtype bf16) only; the %s backend has no "
                         "fp8 coder" % backend)
    if args.code.lower() == "hadamard":
        raise SystemExit("--code hadamard runs on the --backend p2p bf16 engine (--dtype bf16) only; the %s backend has "
                         "no randomized-Hadamard coder" % backend)
    if args.code.lower() == "powersgd":
        raise SystemExit("--code powersgd runs on the --backend p2p bf16 engine (--dtype bf16), which keeps each "
                         "worker's warm state and error-feedback residual; the %s backend's coders keep neither"
                         % backend)
    if args.code.lower() == "sign":
        raise SystemExit("--code sign runs on the --backend p2p bf16 engine (--dtype bf16), which keeps the "
                         "error-feedback residual; scaled sign without it is biased, and the %s backend's coders keep "
                         "none" % backend)
    if args.code.lower() == "signum":
        raise SystemExit("--code signum runs on the --backend p2p bf16 engine (--dtype bf16), which keeps each "
                         "worker's momentum and takes the owners' majority vote; the %s backend's coders keep neither"
                         % backend)
    if args.code.lower() == "dlion":
        raise SystemExit("--code dlion runs on the --backend p2p bf16 engine (--dtype bf16), which keeps each "
                         "worker's Lion momentum and aggregates the signs on the owners; the %s backend's coders keep "
                         "neither" % backend)
    if args.code.lower() == "topk":
        raise SystemExit("--code topk runs on the --backend p2p bf16 engine (--dtype bf16), which keeps the "
                         "error-feedback residual; top-k without it is biased, and the %s backend's coders keep none"
                         % backend)
    if getattr(args, "code_stats", False):
        raise SystemExit("--code-stats reads the statistics of the --backend p2p bf16 engine; the %s backend's "
                         "PyTorch coders do not compute them (run without --code-stats)" % backend)

    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", args.master_addr)
        os.environ.setdefault("MASTER_PORT", str(args.master_port))
        dist.init_process_group(backend, rank=rank, world_size=world)
    if world < 2:
        raise SystemExit("PS training needs world_size >= 2 (1 PS + >=1 worker); use single_machine for 1 process")
    comm = TorchDistTransport()
    comm.enable_backup_rounds(args.num_aggregate)   # same answer on every rank: flag + backend + world size

    train_set, test_set, num_classes = build_datasets(
        args.dataset, args.data_root, synthetic=args.synthetic, seed=args.seed,
        train_len=args.train_len or None, test_len=args.test_len or None)

    if rank == 0:
        master = SyncReplicasMaster_NN(comm=comm, **_kwargs(args, "master"))
        master.build_model(num_classes=num_classes)
        print("I am the master: the world size is {}, cur step: {}".format(master.world_size, master.cur_step))
        master.train()
        print("Done sending messages to workers!")
    else:
        worker = DistributedWorker(comm=comm, **_kwargs(args, "worker"))
        worker.build_model(num_classes=num_classes)
        shard = shard_dataset(train_set, rank - 1, world - 1, seed=args.seed)
        train_loader = DataLoader(shard, batch_size=args.batch_size, shuffle=True, seed=args.seed + rank,
                                  drop_last=True, prefetch=0)
        test_loader = torch.utils.data.DataLoader(test_set, batch_size=args.test_batch_size, shuffle=False)
        print("I am worker: {} in all {} workers, next step: {}".format(worker.rank, worker.world_size - 1, worker.next_step))
        worker.train(train_loader=train_loader, test_loader=test_loader)
        print("Worker Done Jobs! ...")
    if comm.backup_rounds:
        # STOP/bye already synchronised everyone; a collective barrier would hang on a lost worker
        if not comm.clean_shutdown:          # a receive on a dead worker's connection is still pending
            sys.stdout.flush()
            sys.stderr.flush()
            os._exit(0)
    else:
        dist.barrier()
    dist.destroy_process_group()


def _spawn_entry(local_rank: int, args, nproc: int):
    os.environ["RANK"] = str(local_rank)
    os.environ["LOCAL_RANK"] = str(local_rank)
    os.environ["WORLD_SIZE"] = str(nproc)
    os.environ["MASTER_ADDR"] = args.master_addr
    os.environ["MASTER_PORT"] = str(args.master_port)
    run_rank(args)


def main(argv=None):
    args = add_fit_args(argparse.ArgumentParser(description="atomo_b200 distributed PS trainer"), argv)
    if args.nproc and "RANK" not in os.environ:
        import torch.multiprocessing as mp
        attempt = 0
        while True:
            try:
                mp.spawn(_spawn_entry, args=(args, args.nproc), nprocs=args.nproc, join=True)
                break
            except Exception as e:  # a rank raised or exited non-zero (e.g. the PS stopped the job: a worker is gone)
                attempt += 1
                if attempt > args.max_restarts:
                    raise
                # checkpoint/resume-based recovery (SURVEY 5.3/5.4: the reference has neither): the PS state
                # (weights, optimizer, step, LR schedule) comes back from model_step_<N> + its _optim sidecar,
                # workers get parameters from the PS at every step anyway
                print("launcher: job failed ({}); restart {}/{} from the latest checkpoint in {}".format(
                    str(e).strip().splitlines()[0][:120], attempt, args.max_restarts, args.train_dir), flush=True)
                args.resume = True
                args.master_port += 1          # the old rendezvous port may still be in TIME_WAIT
    else:
        run_rank(args)


if __name__ == "__main__":
    main()
