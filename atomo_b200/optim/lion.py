"""Lion (Chen et al. 2023, "Symbolic Discovery of Optimization Algorithms") with the external-gradient API of
:class:`Adam`.

The rule the bf16 engine's parameter server runs (``ShadowEngine(optimizer="lion")``: the decay pass of
``csrc/v2_ema.cu``, then the Lion instantiation of the code's PS kernel), and the oracle its tests compare against.
For every parameter, with ``g`` the averaged gradient and ``m`` its one state tensor (zero at the start):

* ``w <- w * (1 - lr * wd)`` for weights (2 or more dimensions) only: the decoupled decay, as in AdamW
* ``c = b1 * m + (1 - b1) * g``
* ``w <- w - lr * sign(c)``
* ``m <- b2 * m + (1 - b2) * g``

There is no bias correction.  ``sign`` is ``torch.sign`` except that a NaN ``c`` stays NaN (``torch.sign`` maps NaN
to 0, which would freeze the weight and hide the bad gradient).  As on the device, ``lr``, ``b1``, ``b2``,
``1 - b1`` and ``1 - b2`` are fp32 numbers (the last two formed in fp32), the decay factor is ``1 - lr * wd`` in
double rounded to fp32 once, and every multiply and add is its own rounded torch op.  Computed in the dtype of the
parameters.
"""
from __future__ import annotations

import math
from typing import Sequence

import numpy as np
import torch
from torch.optim.optimizer import Optimizer

from .sgd import _as_tensor


def lion_sign(c: torch.Tensor) -> torch.Tensor:
    """+1, -1, 0 for +-0, NaN for NaN."""
    return torch.where(torch.isnan(c), c, torch.sign(c))


class Lion(Optimizer):
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0.0):
        if not lr >= 0.0 or not all(isinstance(b, (int, float)) and 0.0 <= b < 1.0 for b in betas) or len(betas) != 2:
            raise ValueError("Lion: lr must be >= 0 and both betas in [0, 1) (got lr=%r, betas=%r)" % (lr, betas))
        if not 0.0 <= weight_decay < math.inf:
            raise ValueError("Lion: weight_decay must be finite and >= 0 (got %r)" % (weight_decay,))
        super().__init__(params, dict(lr=lr, betas=tuple(float(b) for b in betas), weight_decay=weight_decay))

    def set_lr(self, lr: float) -> None:
        for group in self.param_groups:
            group["lr"] = lr

    @torch.no_grad()
    def step(self, grads: Sequence = None, closure=None, cuda: bool = False):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        grads = list(grads) if grads is not None else None
        offset = 0
        f32 = np.float32
        for group in self.param_groups:
            (b1, b2), lr, wd = group["betas"], group["lr"], group["weight_decay"]
            b1f, b2f, lrf = float(f32(b1)), float(f32(b2)), float(f32(lr))
            om1, om2 = float(f32(1) - f32(b1)), float(f32(1) - f32(b2))
            for p in group["params"]:
                g = p.grad if grads is None else _as_tensor(grads[offset], p)
                offset += 1
                if g is None:
                    continue
                state = self.state[p]
                if len(state) == 0:
                    state["exp_avg"] = torch.zeros_like(p)
                m = state["exp_avg"]
                if p.dim() >= 2 and wd != 0:
                    p.mul_(float(f32(1.0 - float(lr) * wd)))
                c = torch.add(m * b1f, g * om1)
                p.sub_(lion_sign(c) * lrf)
                m.copy_(torch.add(m * b2f, g * om2))
        return loss
