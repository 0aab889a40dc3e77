"""Fused training-mode BatchNorm (+ residual) (+ ReLU) for NHWC bf16 activations.

``BNAct`` is a drop-in ``nn.BatchNorm2d`` (same parameters / buffers / state_dict keys) whose
``forward(x, residual=None, relu=False)`` computes ``relu(bn(x) + residual)``.  With ``fused=True``,
in training mode, on a CUDA bf16 channels_last input it runs the two-pass kernels of
``csrc/bn_kernels.cu`` (statistics, then normalise+add+ReLU in one sweep; backward: reductions, then
dx and the residual gradient in one sweep) instead of PyTorch's four BN kernels plus separate add and
ReLU kernels.  Everything else falls back to the stock ops (identical semantics).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ._ext import load as _load


class _FusedBNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, residual, relu, eps, momentum, acc_fwd, acc_bwd,
                grad_sink=None):
        C = _load()
        y = torch.empty_like(x, memory_format=torch.channels_last)
        nch = x.size(1)
        # acc_* are slices of a per-model arena (the kernels overwrite them with the layer's sums); without an
        # arena (stand-alone use) each call uses its own scratch
        acc = acc_fwd if acc_fwd is not None else torch.empty(2 * nch, dtype=torch.float32, device=x.device)
        mean = torch.empty(nch, dtype=torch.float32, device=x.device)
        invstd = torch.empty(nch, dtype=torch.float32, device=x.device)
        C.bn_forward(x, residual, y, acc, weight, bias, mean, invstd, running_mean, running_var, eps, momentum, relu)
        ctx.save_for_backward(x, y, weight, mean, invstd)
        ctx.relu = relu
        ctx.has_res = residual is not None
        ctx.acc_bwd = acc_bwd
        ctx.grad_sink = grad_sink
        return y

    @staticmethod
    def backward(ctx, dy):
        C = _load()
        x, y, weight, mean, invstd = ctx.saved_tensors
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        nch = x.size(1)
        dx = torch.empty_like(x, memory_format=torch.channels_last)
        dres = torch.empty_like(x, memory_format=torch.channels_last) if ctx.has_res else None
        acc = ctx.acc_bwd if ctx.acc_bwd is not None else torch.empty(2 * nch, dtype=torch.float32, device=x.device)
        if ctx.grad_sink is not None:
            # the engine owns the gradient buffers: dgamma / dbeta are written in place by the kernel and autograd
            # sees no gradient for weight / bias (no AccumulateGrad add kernels for the 2 x #BN vectors)
            dgamma, dbeta = ctx.grad_sink
            C.bn_backward(dy, x, y, dx, dres, mean, invstd, weight, acc, dgamma, dbeta, ctx.relu)
            return dx, None, None, None, None, dres, None, None, None, None, None, None
        dgamma = torch.empty(nch, dtype=torch.float32, device=x.device)
        dbeta = torch.empty(nch, dtype=torch.float32, device=x.device)
        C.bn_backward(dy, x, y, dx, dres, mean, invstd, weight, acc, dgamma, dbeta, ctx.relu)
        return dx, dgamma, dbeta, None, None, dres, None, None, None, None, None, None


class BNAct(nn.BatchNorm2d):
    """BatchNorm2d with an optional fused residual-add and ReLU."""

    fused = False
    _acc_fwd = None   # slices of the per-model statistics arena (see enable_fused_bn)
    _acc_bwd = None
    _grad_sink = None  # (dgamma, dbeta) views the fused backward writes directly (set by the engine)

    def _can_fuse(self, x: torch.Tensor, residual: Optional[torch.Tensor]) -> bool:
        if not (self.fused and self.training and x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4):
            return False
        if x.size(1) % 8 != 0 or x.size(1) > 2048 or not self.track_running_stats or self.momentum is None:
            return False
        if not x.is_contiguous(memory_format=torch.channels_last):
            return False
        if residual is not None and (residual.dtype != x.dtype or residual.shape != x.shape or
                                     not residual.is_contiguous(memory_format=torch.channels_last)):
            return False
        return self.weight is not None and self.weight.dtype == torch.float32

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None, relu: bool = False) -> torch.Tensor:
        if self._can_fuse(x, residual):
            # num_batches_tracked is only consumed when momentum is None (cumulative average), which the
            # fused path does not take: skipping the per-layer counter kernel saves ~20 launches per step
            return _FusedBNFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var, residual,
                                    relu, self.eps, self.momentum, self._acc_fwd, self._acc_bwd, self._grad_sink)
        out = super().forward(x)
        if residual is not None:
            out = out + residual
        return F.relu(out) if relu else out


def enable_fused_bn(module: nn.Module, enabled: bool = True, arena_device=None):
    """Switch every ``BNAct`` of ``module`` to the fused kernels.

    Returns ``(count, arena)``.  With ``arena_device`` one fp32 scratch tensor holds the per-channel
    reduction accumulators of every layer (forward and backward halves); the kernels overwrite a layer's
    slice with its sums, so it needs no zeroing.
    """
    mods = [m for m in module.modules() if isinstance(m, BNAct)]
    arena = None
    if enabled and arena_device is not None and mods:
        total = sum(4 * m.num_features for m in mods)
        arena = torch.zeros(total, dtype=torch.float32, device=arena_device)
        off = 0
        for m in mods:
            c2 = 2 * m.num_features
            m._acc_fwd, m._acc_bwd = arena[off:off + c2], arena[off + c2:off + 2 * c2]
            off += 2 * c2
    for m in mods:
        m.fused = enabled
        if arena is None:
            m._acc_fwd = m._acc_bwd = None
    return len(mods), arena
