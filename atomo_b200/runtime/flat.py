"""Flat parameter / gradient buffers.

The reference moves every parameter tensor separately (P broadcasts, P sends
per step).  Here all parameters of a model live in ONE contiguous fp32 buffer
(each tensor 128-byte aligned) and ``nn.Parameter.data`` / ``.grad`` are views
into it, so a broadcast is one transfer, the PS update is one kernel, and on
the H100 path the buffer can sit in the symmetric NVLink heap with zero copies.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

ALIGN_ELEMS = 32  # 128 bytes of fp32


class FlatLayout:
    def __init__(self, shapes: Sequence[Sequence[int]]):
        self.shapes = [tuple(int(d) for d in s) for s in shapes]
        self.numels, self.offsets = [], []
        off = 0
        for s in self.shapes:
            n = 1
            for d in s:
                n *= d
            self.numels.append(n)
            self.offsets.append(off)
            off += (n + ALIGN_ELEMS - 1) // ALIGN_ELEMS * ALIGN_ELEMS
        self.total = max(off, ALIGN_ELEMS)

    @classmethod
    def from_module(cls, module: torch.nn.Module) -> "FlatLayout":
        return cls([p.shape for p in module.parameters()])

    def views(self, flat: torch.Tensor) -> List[torch.Tensor]:
        return [flat[o:o + n].view(s) for o, n, s in zip(self.offsets, self.numels, self.shapes)]

    def __len__(self):
        return len(self.shapes)


def bind_parameters(module: torch.nn.Module, flat: torch.Tensor, layout: Optional[FlatLayout] = None,
                    copy: bool = True) -> List[torch.Tensor]:
    """Re-home ``module``'s parameters inside ``flat`` (keeping their values)."""
    layout = layout or FlatLayout.from_module(module)
    views = layout.views(flat)
    with torch.no_grad():
        for p, v in zip(module.parameters(), views):
            if copy:
                v.copy_(p.data.to(v.device))
            p.data = v
    return views


def bind_gradients(module: torch.nn.Module, flat_grad: torch.Tensor, layout: Optional[FlatLayout] = None):
    """Make every ``p.grad`` a view into ``flat_grad`` (autograd then accumulates in place)."""
    layout = layout or FlatLayout.from_module(module)
    views = layout.views(flat_grad)
    for p, v in zip(module.parameters(), views):
        p.grad = v
    return views
