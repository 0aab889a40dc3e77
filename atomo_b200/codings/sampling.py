"""Atom-sampling primitives shared by every ATOMO coder.

ATOMO (``/root/reference/README.md:5-7``): given an atomic decomposition
``g = sum_i lambda_i a_i`` and a sparsity budget ``s``, keep atom ``i`` with
probability ``p_i`` and rescale by ``1/p_i`` -> unbiased estimate with
``E[#atoms] = sum_i p_i <= s``.

Two probability rules are provided:

* ``"reference"`` — what the reference implements
  (``src/codings/svd.py:49-67``): ``p = s*lambda/sum(lambda)`` followed by a
  *single* clip to 1 (so ``E[#atoms] <= s``); ``rank == 0`` means
  ``p = lambda/lambda_0``.
* ``"waterfill"`` — the paper's variance-optimal rule: iteratively pin atoms
  whose probability would exceed 1 and redistribute the leftover budget, so
  ``sum_i p_i == min(s, #nonzero atoms)`` exactly.

Two sampling schemes:

* ``"bernoulli"`` — independent coin flips (reference behaviour, variable
  message length, resample when nothing is selected).
* ``"systematic"`` — systematic (stratified-cumulative) sampling: atom ``i`` is
  kept iff an integer lies in ``(c_{i-1}+u, c_i+u]`` with ``c`` the cumulative
  probabilities and a single ``u ~ U[0,1)``.  Marginal inclusion probability is
  exactly ``p_i`` (so the estimator stays unbiased) and the number of kept
  atoms is ``floor``/``ceil`` of ``sum p`` — *fixed-length messages*, which is
  what lets the H100 path use static peer-memory slots and CUDA graphs.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

_TINY = 1e-6  # same degenerate-spectrum threshold as svd.py:50


def atom_probabilities(weights: torch.Tensor, budget: float, rule: str = "reference") -> torch.Tensor:
    """Inclusion probabilities for atoms with non-negative ``weights``.

    ``weights`` is 1-D (singular values or |g_i|).  ``budget`` is the expected
    number of kept atoms ``s``; ``budget == 0`` selects the reference's
    ``p = w / w[0]`` convention (``svd.py:52``) — for unsorted weights we use
    ``w / max(w)``.
    """
    w = weights.detach().to(torch.float64).clamp_min(0)
    if w.numel() == 0:
        return w.to(weights.dtype)
    total = w.sum()
    if float(total) <= 0.0:
        return torch.zeros_like(w).to(weights.dtype)
    if budget == 0:
        p = w / w.max()
        return p.clamp(max=1.0).to(weights.dtype)
    if rule == "reference":
        p = (budget * w / total).clamp(max=1.0)
        return p.to(weights.dtype)
    if rule != "waterfill":
        raise ValueError("unknown probability rule %r" % rule)
    # Iterative water-filling: atoms with budget*w/total >= 1 are pinned to 1.
    nz = int((w > 0).sum())
    s = float(min(budget, nz))
    p = torch.zeros_like(w)
    active = w > 0
    pinned = torch.zeros_like(active)
    for _ in range(w.numel() + 1):
        free = active & ~pinned
        remaining = s - float(pinned.sum())
        denom = w[free].sum()
        if remaining <= 0 or float(denom) <= 0:
            break
        cand = remaining * w / denom
        over = free & (cand >= 1.0)
        if not bool(over.any()):
            p = torch.where(free, cand, p)
            break
        pinned = pinned | over
    p = torch.where(pinned, torch.ones_like(p), p)
    return p.clamp(max=1.0).to(weights.dtype)


def sample_atoms(
    probs: torch.Tensor,
    scheme: str = "bernoulli",
    generator: Optional[torch.Generator] = None,
    uniforms: Optional[torch.Tensor] = None,
    max_atoms: Optional[int] = None,
    max_tries: int = 64,
    allow_empty: bool = False,
) -> torch.Tensor:
    """Return the (sorted) indices of the kept atoms.

    ``allow_empty=True`` accepts a draw that keeps nothing (the unbiased choice: the reference's redraw-until-
    non-empty, svd.py:65-66, over-weights small budgets; the sm_90a engine does not redraw either).

    ``uniforms`` (same length as ``probs`` for bernoulli, length >= 1 for
    systematic) overrides the RNG — the CUDA kernels accept the same override
    so kernel and oracle can be compared bit-for-bit.
    """
    p = probs.detach().to(torch.float64).cpu()
    n = p.numel()
    if n == 0:
        return torch.zeros(0, dtype=torch.long)
    if scheme == "bernoulli":
        for attempt in range(max_tries):
            if uniforms is not None and attempt == 0:
                u = uniforms.detach().to(torch.float64).cpu()[:n]
            else:
                u = torch.rand(n, generator=generator, dtype=torch.float64)
            keep = u < p
            cnt = int(keep.sum())
            # reference: resample when nothing was selected (svd.py:65-66);
            # the fixed-slot GPU path additionally resamples on overflow.
            if cnt == 0 and float(p.max()) > 0 and not allow_empty:
                continue
            if max_atoms is not None and cnt > max_atoms:
                continue
            return torch.nonzero(keep).flatten()
        # pathological: fall back to the most probable atoms
        k = 1 if max_atoms is None else max_atoms
        return torch.sort(torch.topk(p, min(k, n)).indices).values
    if scheme == "systematic":
        if uniforms is not None:
            u = float(uniforms.flatten()[0])
        else:
            u = float(torch.rand(1, generator=generator, dtype=torch.float64))
        c = torch.cumsum(p, 0)
        hi = torch.floor(c + u)
        lo = torch.floor(torch.cat([torch.zeros(1, dtype=torch.float64), c[:-1]]) + u)
        keep = hi > lo
        return torch.nonzero(keep).flatten()
    raise ValueError("unknown sampling scheme %r" % scheme)


def expected_atoms(probs: torch.Tensor) -> float:
    return float(probs.sum())
