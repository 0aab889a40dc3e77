"""Top-k sparsification: the ``k`` largest-magnitude entries of a tensor, sent exactly.

The contractive entry-wise code that error feedback needs (Stich et al. 2018, "Sparsified SGD with memory"; Lin et
al. 2018, Deep Gradient Compression): nothing is rescaled, so ``||A - topk(A)||^2 <= (1 - k_eff / nnz) ||A||^2`` and a
residual fed back step after step stays bounded.  Without error feedback the code is biased.

This coder is the oracle of the bf16 engine's top-k units (``csrc/v2_topk.cu``), applied to the physical-order bf16
vector of a weight tensor:

* ``k = floor(s)`` with ``s = EntryWise(budget).atoms_for(numel)`` (a fraction of numel below 1, else an atom count;
  ``s >= 1``), so top-k never sends more atoms than entry-wise ATOMO expects to send at the same budget;
* magnitudes are compared on the bf16 bits ``bits & 0x7fff`` (exact for finite values, subnormals included); entries
  of magnitude 0 are never kept;
* ``k_eff = min(k, nnz)`` entries are kept: every entry above the threshold magnitude ``T``, then entries equal to
  ``T`` in increasing element order;
* a tensor with an Inf or NaN keeps nothing;
* no random numbers: the kept set depends only on the bf16 values.
"""
from __future__ import annotations

import math

import torch

from .coding import Coding, register
from .entrywise import EntryWise


def bf16_magnitude_bits(flat: torch.Tensor) -> torch.Tensor:
    """``bits & 0x7fff`` of the bf16 rounding of ``flat``, as int32."""
    return flat.reshape(-1).to(torch.bfloat16).view(torch.int16).to(torch.int32) & 0x7FFF


@register("topk")
class TopK(Coding):
    def __init__(self, budget: float = 0.05, *args, **kwargs):
        super().__init__()
        if not budget > 0:
            raise ValueError("budget must be positive (a fraction of numel below 1, else an atom count)")
        self.budget = float(budget)

    def k_for(self, numel: int) -> int:
        return int(math.floor(EntryWise(self.budget).atoms_for(numel)))

    def select(self, flat: torch.Tensor) -> torch.Tensor:
        """Sorted element indices (int64) of the kept entries of a flat tensor (bf16-rounded first)."""
        mag = bf16_magnitude_bits(flat)
        if bool((mag >= 0x7F80).any()):                   # exponent all ones: Inf / NaN keeps nothing
            return torch.zeros(0, dtype=torch.long, device=flat.device)
        k_eff = min(self.k_for(mag.numel()), int((mag != 0).sum()))
        order = torch.sort(-mag, stable=True).indices     # descending magnitude, ties in element order
        return torch.sort(order[:k_eff]).values

    def encode(self, grad: torch.Tensor, **kwargs) -> dict:
        shape = list(grad.shape)
        flat = grad.detach().reshape(-1)
        idx = self.select(flat)
        val = flat.to(torch.bfloat16).to(torch.float32)[idx]
        return {"idx": idx.to(torch.int32), "val": val, "shape": shape, "numel": flat.numel()}

    def decode(self, code: dict, cuda: bool = False, **kwargs) -> torch.Tensor:
        out = torch.zeros(int(code["numel"]), dtype=torch.float32, device=code["val"].device)
        out[code["idx"].to(torch.long)] = code["val"]
        out = out.reshape(code["shape"])
        return out.cuda() if cuda else out
