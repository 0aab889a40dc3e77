"""Evaluator CLI (parity: ``/root/reference/src/distributed_evaluator.py:45-54,
136-160``): ``--eval-batch-size --eval-freq --model-dir --dataset --network``."""
import argparse

import torch

from .data import build_datasets
from .runtime.evaluator import DistributedEvaluator
from .utils.flags import bool_flag


def main(argv=None):
    ap = argparse.ArgumentParser(description="atomo_b200 checkpoint-polling evaluator")
    ap.add_argument("--eval-batch-size", type=int, default=10000)
    ap.add_argument("--eval-freq", type=int, default=50)
    ap.add_argument("--model-dir", type=str, default="output/models/")
    ap.add_argument("--dataset", type=str, default="MNIST")
    ap.add_argument("--network", type=str, default="LeNet")
    ap.add_argument("--synthetic", type=bool_flag, default=None)
    ap.add_argument("--data-root", type=str, default=".")
    ap.add_argument("--test-len", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--max-evals", type=int, default=0, help="stop after N evaluations (0 = forever)")
    ap.add_argument("--timeout", type=float, default=0.0, help="stop after this many idle seconds (0 = never)")
    ap.add_argument("--poll-seconds", type=float, default=10.0)
    ap.add_argument("--ema", type=bool_flag, default=False,
                    help="evaluate the weight average model_step_<N>_ema (--ema-decay) instead of model_step_<N>")
    args = ap.parse_args(argv)
    _, test, ncls = build_datasets(args.dataset, args.data_root, args.synthetic, args.seed, None, args.test_len or None)
    loader = torch.utils.data.DataLoader(test, batch_size=args.eval_batch_size, shuffle=False)
    device = "cuda" if torch.cuda.is_available() else "cpu"
    ev = DistributedEvaluator(model_dir=args.model_dir, eval_freq=args.eval_freq, network=args.network,
                              dataset=args.dataset, num_classes=ncls, device=device,
                              eval_batch_size=args.eval_batch_size, poll_seconds=args.poll_seconds, ema=args.ema)
    return ev.evaluate(loader, max_evals=args.max_evals or None, timeout=args.timeout or None)


if __name__ == "__main__":
    main()
