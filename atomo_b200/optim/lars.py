"""Layer-wise adaptive rate scaling (LARS, You et al. 2017) with the external-gradient API of :class:`SGD`.

The rule the bf16 engine's parameter server runs (``csrc/v2_layerwise.cu``), and the oracle its tests compare
against.  For every weight (a parameter with 2 or more dimensions), with ``g`` the averaged gradient:

* ``d = g + wd * w``
* ``ratio = eta * ||w|| / (||g|| + wd * ||w||)``, ``1`` when ``||w|| == 0`` or the denominator is ``0``
* ``m = mu * m + ratio * d`` (``m = ratio * d`` on the first step), ``w -= lr * m``

1-D parameters (BN, biases) take plain momentum SGD without weight decay and trust ratio.  Computed in the dtype of
the parameters: in fp64 when given fp64 tensors.
"""
from __future__ import annotations

from typing import Sequence

import torch
from torch.optim.optimizer import Optimizer

from .sgd import _as_tensor


def trust_ratio(num: torch.Tensor, den: torch.Tensor, wn: torch.Tensor) -> torch.Tensor:
    """``num / den``, or 1 where ``||w||`` or the denominator is 0 (as a 0-d tensor of ``num``'s dtype)."""
    ok = bool(wn > 0) and bool(den > 0)
    return num / den if ok else torch.ones((), dtype=num.dtype, device=num.device)


class LARS(Optimizer):
    def __init__(self, params, lr=0.1, momentum=0.0, weight_decay=0.0, trust_coefficient=0.001, nesterov=False,
                 dampening=0.0):
        if lr < 0.0 or momentum < 0.0 or weight_decay < 0.0 or trust_coefficient <= 0.0:
            raise ValueError("LARS: lr, momentum and weight_decay must be >= 0 and trust_coefficient > 0")
        if nesterov or dampening != 0:
            raise ValueError("LARS takes plain momentum: no nesterov, dampening 0")
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay,
                                      trust_coefficient=trust_coefficient))

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
        for group in self.param_groups:
            lr, mu, wd, eta = group["lr"], group["momentum"], group["weight_decay"], group["trust_coefficient"]
            for p in group["params"]:
                g = p.grad if grads is None else _as_tensor(grads[offset], p)
                offset += 1
                if g is None:
                    continue
                state = self.state[p]
                if p.dim() >= 2:
                    d = g.add(p, alpha=wd)
                    wn, gn = p.norm(), g.norm()
                    ratio = trust_ratio(eta * wn, gn + wd * wn, wn)
                    state["ratio"] = float(ratio)
                    x = d * ratio
                else:
                    x = g
                if mu == 0 and p.dim() < 2:
                    p.add_(x, alpha=-lr)
                    continue
                if "momentum_buffer" not in state:
                    buf = state["momentum_buffer"] = x.clone()
                else:
                    buf = state["momentum_buffer"].mul_(mu).add_(x)
                p.add_(buf, alpha=-lr)
        return loss
