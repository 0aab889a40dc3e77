#!/usr/bin/env python
"""How much variance does cutting square-ish tensors into 32-column blocks cost (or save) against the reference's
whole-tensor spectral coder?  For real gradients (one backward pass of the named network on synthetic data) and every
matrix-shaped parameter, estimate the relative variance E||decode - g||^2 / ||g||^2 and the bytes on the wire of

  svd  r   whole-tensor SVD atoms (reference estimator, needs a full SVD of the matrix per step)
  bsvd r   the sm_90a engine's estimator (3x3 convs whole; fc / 1x1 layers in <= 32-column blocks)

    python scripts/variance_study.py --network ResNet18 --rank 3 --out docs/experiments/variance_resnet18.md
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from atomo_b200 import codings                             # noqa: E402
from atomo_b200.codings.block_svd import unit_table        # noqa: E402
from atomo_b200.data import SyntheticImageDataset          # noqa: E402
from atomo_b200.models import build_model, input_shape     # noqa: E402


def rel_var(coder, g, draws):
    tot, nbytes = 0.0, 0
    for _ in range(draws):
        code = coder.encode(g)
        nbytes += codings.Coding.wire_bytes(code)
        tot += float((coder.decode(code).reshape(g.shape) - g).pow(2).sum())
    return tot / draws / float(g.pow(2).sum()), nbytes / draws


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--network", default="ResNet18")
    ap.add_argument("--dataset", default="")
    ap.add_argument("--rank", type=int, default=3)
    ap.add_argument("--draws", type=int, default=40)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    torch.manual_seed(0)
    torch.set_num_threads(6)
    ds = args.dataset or ("MNIST" if args.network in ("LeNet", "FC") else "Cifar10")
    shape = input_shape(args.network, ds)
    model = build_model(args.network, 10, ds)
    x, y = SyntheticImageDataset(shape, 10, 4096, seed=0, noise=2.0).materialize(args.batch_size)
    F.cross_entropy(model(x), y).backward()
    gen = torch.Generator().manual_seed(1)
    svd = codings.build("svd", rank=args.rank, generator=gen)
    bsvd = codings.build("bsvd", rank=args.rank, generator=gen)
    bglob = codings.build("bsvd", rank=args.rank, generator=gen, allocation="global")
    rows, tot = [], {"dense": 0, "svd_b": 0, "bsvd_b": 0, "svd_v": 0.0, "bsvd_v": 0.0, "g2": 0.0, "glob_b": 0, "glob_v": 0.0}
    for name, p in model.named_parameters():
        if p.dim() < 2:
            continue
        g = p.grad.detach().float()
        kinds = unit_table(tuple(g.shape), args.rank)
        vs, bs = rel_var(svd, g, args.draws)
        vb, bb = rel_var(bsvd, g, args.draws) if kinds[0][0] != "dense" else (0.0, g.numel() * 4)
        vg, bg = rel_var(bglob, g, args.draws) if kinds[0][0] != "dense" else (0.0, g.numel() * 4)
        g2 = float(g.pow(2).sum())
        tot["glob_b"] += bg; tot["glob_v"] += vg * g2
        tot["dense"] += g.numel() * 4; tot["svd_b"] += bs; tot["bsvd_b"] += bb
        tot["svd_v"] += vs * g2; tot["bsvd_v"] += vb * g2; tot["g2"] += g2
        if kinds[0][0] != "slab":        # the interesting rows: tensors the two estimators treat differently
            rows.append((name, tuple(g.shape), kinds[0][0] + (" x%d" % len(kinds) if kinds[0][0] == "block" else ""),
                         vs, bs, vb, bb, vg, bg))
    lines = ["# Block-spectral vs whole-tensor spectral estimator: %s, rank budget %d, %d draws per tensor"
             % (args.network, args.rank, args.draws), "",
             "Relative variance = E||decode - g||^2 / ||g||^2 of one worker's estimate (real gradients of one backward pass;",
             "`scripts/variance_study.py`).  3x3 convolutions are coded identically by both (not listed).", "",
             "`bsvd global` = the same blocks with ONE budget per tensor (p_i = min(1, r sigma_i / sum of all blocks' sigma)): a",
             "candidate for the next kernel revision, CPU oracle only.", "",
             "| tensor | shape | bf16-engine units | svd: rel. variance | svd: bytes | bsvd: rel. variance | bsvd: bytes | bsvd global: rel. variance | bsvd global: bytes |",
             "|---|---|---|---|---|---|---|---|---|"]
    for name, shp, kind, vs, bs, vb, bb, vg, bg in rows:
        lines.append("| `%s` | %s | %s | %.2f | %d | %.2f | %d | %.2f | %d |" % (name, "x".join(map(str, shp)), kind, vs, bs, vb, bb, vg, bg))
    lines += ["", "Whole model (all matrix-shaped tensors, variance weighted by ||g||^2): svd %.2f at %.2f MB, bsvd %.2f at "
              "%.2f MB, bsvd global %.2f at %.2f MB (dense: %.2f MB)."
              % (tot["svd_v"] / tot["g2"], tot["svd_b"] / 2 ** 20, tot["bsvd_v"] / tot["g2"], tot["bsvd_b"] / 2 ** 20,
                 tot["glob_v"] / tot["g2"], tot["glob_b"] / 2 ** 20, tot["dense"] / 2 ** 20)]
    text = "\n".join(lines) + "\n"
    print(text)
    if args.out:
        open(args.out, "w").write(text)


if __name__ == "__main__":
    main()
