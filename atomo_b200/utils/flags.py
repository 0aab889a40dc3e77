"""Launcher flag surface (parity: ``add_fit_args``,
``/root/reference/src/distributed_nn.py:31-82`` — every flag of SURVEY.md 2.7 is
kept with its default) plus the H100-specific additions."""
from __future__ import annotations

import argparse


def bool_flag(v) -> bool:
    """The reference declares ``type=bool`` (any non-empty string is True and
    the scripts pass ``--enable-gpu=`` for False).  This keeps that contract
    and additionally understands 0/false/no."""
    if isinstance(v, bool):
        return v
    return str(v).strip().lower() not in ("", "0", "false", "no", "off", "none")


def add_fit_args(parser: argparse.ArgumentParser, argv=None):
    p = parser
    p.add_argument("--batch-size", type=int, default=128, metavar="N")
    p.add_argument("--test-batch-size", type=int, default=1000, metavar="N")
    p.add_argument("--max-steps", type=int, default=10000, metavar="N")
    p.add_argument("--epochs", type=int, default=100, metavar="N")
    p.add_argument("--lr", type=float, default=0.01, metavar="LR")
    p.add_argument("--momentum", type=float, default=0.5, metavar="M")
    p.add_argument("--lr-shrinkage", type=float, default=0.95, metavar="M")
    p.add_argument("--no-cuda", action="store_true", default=False)
    p.add_argument("--seed", type=int, default=1, metavar="S")
    p.add_argument("--log-interval", type=int, default=10, metavar="N")
    p.add_argument("--network", type=str, default="LeNet", metavar="N")
    p.add_argument("--code", type=str, default="sgd",
                   help="sgd | svd | qsgd | terngrad | entrywise | qsvd | bsvd (block-spectral: the estimator the sm_90a "
                        "bf16 engine applies under --code svd, as a plain PyTorch coder) | topk (the --entry-budget "
                        "largest entries per tensor, sent exactly; --backend p2p --dtype bf16 only, meant for "
                        "--error-feedback 1) | sign (scaled sign: one bit per element and one fp32 scale "
                        "||b||_1/|b| per --bucket-size bucket, a multiple of 64 in [64, 4096]; --backend p2p --dtype "
                        "bf16 only, meant for --error-feedback 1) | powersgd (rank --svd-rank in [1, 4] factors of every "
                        "weight matrix from one warm-started power step; --backend p2p --dtype bf16 only, meant for "
                        "--error-feedback 1) | fp8 (one e4m3 byte per element, stochastically rounded and so "
                        "unbiased, and one power-of-two fp32 scale per --bucket-size bucket, a multiple of 64 in "
                        "[64, 4096]; --backend p2p --dtype bf16 only)")
    p.add_argument("--bucket-size", type=int, default=512)
    p.add_argument("--dataset", type=str, default="MNIST", metavar="N")
    p.add_argument("--comm-type", type=str, default="Bcast", metavar="N")
    p.add_argument("--num-aggregate", type=int, default=0, metavar="N",
                   help="gradients to wait for per step (0 = all workers; reference default 5 was a no-op).  N < workers = "
                        "backup workers: the PS never waits for a straggler and keeps training when a worker is lost")
    p.add_argument("--eval-freq", type=int, default=50, metavar="N")
    p.add_argument("--train-dir", type=str, default="output/models/", metavar="N")
    p.add_argument("--compress", type=bool_flag, default=False)
    p.add_argument("--enable-gpu", type=bool_flag, default=False)
    p.add_argument("--svd-rank", type=int, default=0)
    p.add_argument("--quantization-level", type=int, default=4)
    # ---- additions -----------------------------------------------------
    p.add_argument("--backend", type=str, default="auto", choices=["auto", "gloo", "nccl", "p2p"],
                   help="gloo (CPU), nccl (baseline), p2p (fused NVLink peer-memory engine)")
    p.add_argument("--nproc", type=int, default=0, help="spawn this many local ranks (0 = use torchrun env)")
    p.add_argument("--synthetic", type=bool_flag, default=None, help="force synthetic data (default: auto)")
    p.add_argument("--data-root", type=str, default=".")
    p.add_argument("--train-len", type=int, default=0, help="truncate the training set (0 = full)")
    p.add_argument("--test-len", type=int, default=0)
    p.add_argument("--entry-budget", type=float, default=0.05, help="entry-wise ATOMO / top-k budget: a fraction of each tensor's "
                   "elements below 1, else an atom count (top-k sends floor of it)")
    p.add_argument("--sampling", type=str, default="bernoulli", choices=["bernoulli", "systematic"])
    p.add_argument("--prob-rule", type=str, default="reference", choices=["reference", "waterfill"])
    p.add_argument("--optimizer", type=str, default="sgd", choices=["sgd", "adam"])
    p.add_argument("--weight-decay", type=float, default=0.0)
    p.add_argument("--nesterov", type=bool_flag, default=False)
    p.add_argument("--resume", type=bool_flag, default=False)
    p.add_argument("--metrics-file", type=str, default="",
                   help="also write every logged step as one JSON object per line to <path>.rank<R>.jsonl")
    p.add_argument("--max-restarts", type=int, default=0,
                   help="--nproc self-spawn: when the job fails (a rank died, the PS stopped it), relaunch it up to N "
                        "times from the latest checkpoint (--resume 1 is implied for the relaunches).  Under torchrun "
                        "use its own --max-restarts together with --resume 1")
    p.add_argument("--dtype", type=str, default="fp32", choices=["fp32", "bf16"])
    p.add_argument("--ps-mode", type=str, default="sharded", choices=["sharded", "colocated", "dedicated"],
                   help="p2p backend: sharded = every GPU trains and owns 1/N of the PS tiles (bf16 engine); "
                        "colocated = rank 0 hosts the whole PS and also trains; dedicated = rank 0 only serves")
    p.add_argument("--engine", type=str, default="auto", choices=["auto", "shadow", "fused"],
                   help="p2p backend: auto = the overlapped sharded bf16 engine for --dtype bf16 with --code "
                        "svd|qsvd|sgd|topk|sign|powersgd|fp8, the fp32-flat engine otherwise; shadow = the bf16 engine (also --code "
                        "qsgd|terngrad, needs --dtype bf16); fused = the fp32-flat engine")
    p.add_argument("--groups", type=int, default=5, help="p2p/bf16: backward groups pushed while backward runs")
    p.add_argument("--shrinkage-freq", type=int, default=50, help="steps between LR shrinkages (reference: 50)")
    p.add_argument("--flag-timeout", type=float, default=120.0,
                   help="p2p: seconds a device-side wait on a peer flag may spin before the sticky error code is set")
    p.add_argument("--straggler-kill", type=bool_flag, default=False,
                   help="with --num-aggregate < workers: layer-wise (split) backward on the workers and a tag-77 kill "
                        "signal from the PS once enough gradients arrived (LeNet / FC / ResNet18 / ResNet34)")
    p.add_argument("--master-addr", type=str, default="127.0.0.1")
    p.add_argument("--master-port", type=int, default=29511)
    p.add_argument("--eval-batches", type=int, default=0, help="cap test batches per evaluation (0 = all)")
    p.add_argument("--gpu-data", type=bool_flag, default=False,
                   help="p2p backend: keep the rank's shard and the test set on the GPU and build every batch there "
                        "(same sample order and augmentation as the CPU loader; not for --dataset ImageNet)")
    p.add_argument("--code-stats", type=bool_flag, default=False,
                   help="p2p backend, bf16 engine: per-layer estimator statistics of the code (expected squared error "
                        "given the gradient, expected / realized atoms, realized push bytes) in every --metrics-file "
                        "record; not for --code qsvd")
    p.add_argument("--error-feedback", type=bool_flag, default=False,
                   help="p2p backend, bf16 engine: every worker keeps the part of its gradient the code did not send "
                        "(an fp32 residual per weight) and adds it to the next step's gradient before coding; --code "
                        "svd | entrywise | topk | qsgd | sign | powersgd | fp8 (it stays bounded with svd top-k, topk, "
                        "sign and powersgd, the contractive codes, and with fp8, whose variance is small), every push counted (no --num-aggregate below the worker "
                        "count).  Residuals (and PowerSGD's warm state) are not checkpointed: --resume starts them afresh")
    return p.parse_args(argv)
