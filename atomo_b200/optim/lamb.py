"""Layer-wise adaptive moments (LAMB, You et al. 2019) with the external-gradient API of :class:`SGD`.

The rule the bf16 engine's parameter server runs (``csrc/v2_layerwise.cu``), and the oracle its tests compare
against.  For every weight (a parameter with 2 or more dimensions), with ``g`` the averaged gradient and ``t`` the
step count:

* ``m = b1 * m + (1 - b1) * g``, ``v = b2 * v + (1 - b2) * g^2`` (the moments of the engine's Adam)
* ``u = (m / bc1) / (sqrt(v) / sqrt(bc2) + eps) + wd * w`` with ``bc = 1 - b^t`` (decoupled weight decay)
* ``ratio = ||w|| / ||u||``, ``1`` when either norm is ``0``; ``w -= lr * ratio * u``

1-D parameters (BN, biases) take the engine's Adam without weight decay and trust ratio:
``w -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)``.  Computed in the dtype of the parameters: in fp64 when given
fp64 tensors.
"""
from __future__ import annotations

import math
from typing import Sequence

import torch
from torch.optim.optimizer import Optimizer

from .lars import trust_ratio
from .sgd import _as_tensor


class LAMB(Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False):
        if lr < 0.0 or weight_decay < 0.0 or not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("LAMB: lr and weight_decay must be >= 0 and betas in [0, 1)")
        if amsgrad:
            raise ValueError("LAMB has no AMSGrad variant")
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

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
            (b1, b2), lr, eps, wd = group["betas"], group["lr"], group["eps"], group["weight_decay"]
            for p in group["params"]:
                g = p.grad if grads is None else _as_tensor(grads[offset], p)
                offset += 1
                if g is None:
                    continue
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p)
                    state["exp_avg_sq"] = torch.zeros_like(p)
                state["step"] += 1
                t = state["step"]
                m, v = state["exp_avg"], state["exp_avg_sq"]
                m.mul_(b1).add_(g, alpha=1 - b1)
                v.mul_(b2).addcmul_(g, g, value=1 - b2)
                bc1, sbc2 = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
                adam = (m / bc1) / (v.sqrt() / sbc2 + eps)
                if p.dim() >= 2:
                    u = adam.add(p, alpha=wd)
                    wn, un = p.norm(), u.norm()
                    ratio = trust_ratio(wn, un, wn)
                    state["ratio"] = float(ratio)
                    p.sub_(u * (lr * ratio))
                else:
                    p.sub_(adam, alpha=lr)
        return loss
