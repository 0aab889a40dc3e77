"""Adam with decoupled weight decay (AdamW, Loshchilov & Hutter 2019) with the external-gradient API of :class:`Adam`.

The rule the bf16 engine's parameter server runs (``ShadowEngine(optimizer="adamw")``: the decay pass of
``csrc/v2_ema.cu``, then the engine's Adam with weight decay 0), and the oracle its tests compare against.  It is
``torch.optim.AdamW`` with two parameter groups, the usual practice.  For every weight (a parameter with 2 or more
dimensions), with ``g`` the averaged gradient and ``t`` the step count:

* ``w <- w * (1 - lr * wd)`` (the decoupled decay, before the moments see the gradient)
* ``m = b1 * m + (1 - b1) * g``, ``v = b2 * v + (1 - b2) * g^2``; AMSGrad: ``v_max = max(v_max, v)`` replaces ``v``
* ``w -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)`` with ``bc = 1 - b^t``

1-D parameters (BN, biases) take the same Adam step without the decay.  Computed in the dtype of the parameters: in
fp64 when given fp64 tensors.
"""
from __future__ import annotations

import math
from typing import Sequence

import torch
from torch.optim.optimizer import Optimizer

from .sgd import _as_tensor


class AdamW(Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False):
        if not lr >= 0.0 or not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError("AdamW: lr must be >= 0 and betas in [0, 1)")
        if not 0.0 <= weight_decay < math.inf:
            raise ValueError("AdamW: weight_decay must be finite and >= 0 (got %r)" % (weight_decay,))
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad))

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
                    if group["amsgrad"]:
                        state["max_exp_avg_sq"] = torch.zeros_like(p)
                state["step"] += 1
                t = state["step"]
                if p.dim() >= 2 and wd != 0:
                    p.mul_(1 - lr * wd)
                m, v = state["exp_avg"], state["exp_avg_sq"]
                m.mul_(b1).add_(g, alpha=1 - b1)
                v.mul_(b2).addcmul_(g, g, value=1 - b2)
                if group["amsgrad"]:
                    torch.maximum(state["max_exp_avg_sq"], v, out=state["max_exp_avg_sq"])
                    v = state["max_exp_avg_sq"]
                bc1, sbc2 = 1 - b1 ** t, math.sqrt(1 - b2 ** t)
                p.addcdiv_(m, v.sqrt().div_(sbc2).add_(eps), value=-lr / bc1)
        return loss
