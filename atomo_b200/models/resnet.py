"""ResNet family, spec-driven.

Capability parity with ``/root/reference/src/model_ops/resnet.py`` (CIFAR-style ResNet: 3x3 stem, no
max-pool, 4x4 average pool, ``BasicBlock`` x [2,2,2,2] ... ``Bottleneck`` x [3,8,36,3]) — every depth
constructs and runs here (the reference's 34/50/101/152 constructors crash, SURVEY.md 2.9) — plus an
ImageNet stem (7x7/2 conv, 3x3/2 max-pool, global average pool) for BASELINE config 4.

A residual block is described by a tuple of ``(kernel, channels, stride)`` conv stages; the module and
parameter names (``conv1, bn1, ..., shortcut.0, shortcut.1``, ``layer1..4``, ``linear``) and therefore the
``parameters()`` order match the reference, so the per-tensor coders see the same 62 tensors for ResNet-18.
Every normalisation layer is a :class:`~atomo_b200.ops.fused_bn.BNAct`: BN + residual add + ReLU is one call
(and one fused sm_90a kernel pair when enabled).
"""
from typing import Sequence, Tuple

import torch.nn as nn
import torch.nn.functional as F

from ..ops.fused_bn import BNAct
from ..ops.split_conv import Conv2d

Stage = Tuple[int, int, int]  # (kernel size, output channels, stride)


class _ResidualBlock(nn.Module):
    expansion = 1

    def __init__(self, in_planes: int, stages: Sequence[Stage], stride: int):
        super().__init__()
        self.depth = len(stages)
        width = in_planes
        for i, (k, ch, s) in enumerate(stages, start=1):
            setattr(self, "conv%d" % i, Conv2d(width, ch, k, s, k // 2, bias=False))
            setattr(self, "bn%d" % i, BNAct(ch))
            width = ch
        self.shortcut = nn.Sequential()  # identity unless the shape changes
        if stride != 1 or in_planes != width:
            self.shortcut = nn.Sequential(Conv2d(in_planes, width, 1, stride, bias=False), BNAct(width))

    def forward(self, x):
        out = x
        for i in range(1, self.depth):
            out = getattr(self, "bn%d" % i)(getattr(self, "conv%d" % i)(out), relu=True)
        last_conv, last_bn = getattr(self, "conv%d" % self.depth), getattr(self, "bn%d" % self.depth)
        return last_bn(last_conv(out), residual=self.shortcut(x), relu=True)  # bn + add + relu in one op


class BasicBlock(_ResidualBlock):
    expansion = 1

    def __init__(self, in_planes, planes, stride=1):
        super().__init__(in_planes, ((3, planes, stride), (3, planes, 1)), stride)


class Bottleneck(_ResidualBlock):
    expansion = 4

    def __init__(self, in_planes, planes, stride=1):
        super().__init__(in_planes, ((1, planes, 1), (3, planes, stride), (1, self.expansion * planes, 1)), stride)


class ResNet(nn.Module):
    widths = (64, 128, 256, 512)

    def __init__(self, block, num_blocks, num_classes=10, imagenet_stem=False):
        super().__init__()
        self.imagenet_stem = imagenet_stem
        self.conv1 = Conv2d(3, 64, 7, 2, 3, bias=False) if imagenet_stem else Conv2d(3, 64, 3, 1, 1, bias=False)
        self.bn1 = BNAct(64)
        self.in_planes = 64
        for idx, (planes, n) in enumerate(zip(self.widths, num_blocks), start=1):
            setattr(self, "layer%d" % idx, self._make_layer(block, planes, n, 1 if idx == 1 else 2))
        self.linear = nn.Linear(self.widths[-1] * block.expansion, num_classes)

    def _make_layer(self, block, planes, n, stride):
        blocks = []
        for s in (stride,) + (1,) * (n - 1):
            blocks.append(block(self.in_planes, planes, s))
            self.in_planes = planes * block.expansion
        return nn.Sequential(*blocks)

    def forward(self, x):
        out = self.bn1(self.conv1(x), relu=True)
        if self.imagenet_stem:
            out = F.max_pool2d(out, 3, 2, 1)
        for idx in range(1, 5):
            out = getattr(self, "layer%d" % idx)(out)
        if self.imagenet_stem:
            out = F.adaptive_avg_pool2d(out, 1)
        elif out.shape[-2:] == (4, 4):
            out = out.mean(dim=(2, 3))          # == avg_pool2d(out, 4) on a 4x4 map; its backward is one broadcast
        else:
            out = F.avg_pool2d(out, 4)
        return self.linear(out.flatten(1))


_DEPTHS = {18: (BasicBlock, (2, 2, 2, 2)), 34: (BasicBlock, (3, 4, 6, 3)), 50: (Bottleneck, (3, 4, 6, 3)),
           101: (Bottleneck, (3, 4, 23, 3)), 152: (Bottleneck, (3, 8, 36, 3))}


def _resnet(depth, num_classes, **kw):
    block, layout = _DEPTHS[depth]
    return ResNet(block, list(layout), num_classes, **kw)


def ResNet18(num_classes=10, **kw): return _resnet(18, num_classes, **kw)
def ResNet34(num_classes=10, **kw): return _resnet(34, num_classes, **kw)
def ResNet50(num_classes=10, **kw): return _resnet(50, num_classes, **kw)
def ResNet101(num_classes=10, **kw): return _resnet(101, num_classes, **kw)
def ResNet152(num_classes=10, **kw): return _resnet(152, num_classes, **kw)
