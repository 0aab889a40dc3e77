"""Convolution whose backward computes the weight gradient on a stream of its own.

Nothing later in the backward reads a convolution's weight gradient: only the gradient coder does, and it runs on a
side stream.  ``Conv2d`` is a drop-in ``nn.Conv2d`` (same parameters and state_dict keys).  With a wgrad stream set
(:func:`enable_split_wgrad`) its backward, ``conv_backward_split`` of the native extension, makes the two calls the
stock autograd node makes as one: ``at::convolution_backward`` for the input gradient on the current stream and for
the weight gradient on the wgrad stream, so the next layer's backward does not wait for the weight gradient.  Both
are the same cuDNN calls with the same algorithm choice, so every value is the same as on the stock path.

Whoever reads a weight gradient on another stream waits for the wgrad stream first (the engine records an event on
it when a gradient group is complete) and calls ``record_stream`` for its stream.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from ._ext import load as _load


class _SplitWgradConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, stride, padding, dilation, groups, wgrad_stream):
        ctx.save_for_backward(x, weight)
        ctx.conf = (stride, padding, dilation, groups)
        ctx.wgrad_stream = wgrad_stream
        return F.conv2d(x, weight, None, stride, padding, dilation, groups)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        stride, padding, dilation, groups = ctx.conf
        # csrc/bindings.cpp conv_backward_split: dgrad here, wgrad on the wgrad stream
        dx, dw = _load().conv_backward_split(dy, x, weight, list(stride), list(padding), list(dilation), groups,
                                             ctx.needs_input_grad[0], ctx.needs_input_grad[1],
                                             ctx.wgrad_stream.cuda_stream)
        return dx, dw, None, None, None, None, None


class Conv2d(nn.Conv2d):
    """nn.Conv2d whose weight gradient runs on ``wgrad_stream`` when one is set (CUDA bf16 input and weight, no
    bias, zero padding); the stock path otherwise."""

    wgrad_stream = None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.wgrad_stream is not None and x.is_cuda and self.weight.dtype == torch.bfloat16 and \
                self.bias is None and self.padding_mode == "zeros" and isinstance(self.padding, tuple):
            if x.dtype == torch.float32 and torch.is_autocast_enabled("cuda") and \
                    torch.get_autocast_dtype("cuda") == torch.bfloat16:
                x = x.to(torch.bfloat16)    # the cast autocast makes (the fp32 network input of the stem)
            if x.dtype == torch.bfloat16:   # the saved tensors are then the ones the convolution read
                return _SplitWgradConvFn.apply(x, self.weight, self.stride, self.padding, self.dilation, self.groups,
                                               self.wgrad_stream)
        return super().forward(x)


def enable_split_wgrad(module: nn.Module, stream=None) -> int:
    """Compute the weight gradient of every ``Conv2d`` of ``module`` on ``stream`` (None: the stock backward).
    Returns the number of layers."""
    mods = [m for m in module.modules() if isinstance(m, Conv2d)]
    for m in mods:
        m.wgrad_stream = stream
    return len(mods)
