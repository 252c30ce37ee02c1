"""CIFAR-style ResNets (3x3 stem, no max-pool, 4x4 average pool, 10 classes).

Architecture parity with the reference (src/model_ops/resnet.py:14-113): BasicBlock (expansion 1) and
Bottleneck (expansion 4) with a conv1x1+BN projection shortcut whenever stride != 1 or the width changes;
all convolutions are bias-free.  Parameter-tensor counts / sizes (checked in tests/test_models.py):
ResNet18 62 / 11,173,962; ResNet34 110 / 21,282,122; ResNet50 161 / 23,520,842; ResNet101 314 / 42,512,970;
ResNet152 467 / 58,156,618.

``num_classes`` is an extension (the reference hard-codes 10); ``imagenet_stem=True`` swaps the 3x3 CIFAR stem for the
7x7 / stride-2 convolution + 3x3 / stride-2 max-pool of the ImageNet ResNets and pools adaptively (used for
ResNet-50 on synthetic 224x224 ImageNet-shaped data).  The defaults reproduce the reference exactly.
"""
from __future__ import annotations

from typing import List, Type

import torch
import torch.nn.functional as F
from torch import nn

from ..ops.conv import Conv2d
from ..ops.linear import Linear
from ..ops.norm import FusedBatchNorm2d
from ..ops.pool import global_avg_pool
from .split import make_split


def _conv(cin: int, cout: int, k: int, stride: int = 1) -> nn.Conv2d:
    # ops.conv.Conv2d is nn.Conv2d whose 1x1 / stride-1 case runs on the wgmma GEMM (bottleneck conv1 / conv3)
    return Conv2d(cin, cout, kernel_size=k, stride=stride, padding=k // 2, bias=False)


def _bn_residual_relu(bn: FusedBatchNorm2d, c: torch.Tensor, seq: nn.Sequential, x: torch.Tensor) -> torch.Tensor:
    """relu(bn(c) + shortcut(x)) for an identity or projection (conv1x1 + BN) shortcut.  The projection's BatchNorm statistics
    come from its convolution too, and ``residual_bn`` lets both BatchNorms run as one pass each way (ops/norm.py)."""
    if len(seq) == 0:
        return bn(c, residual=x, relu=True)
    conv, bn_s = seq[0], seq[1]
    return bn(c, residual_bn=(bn_s, conv(x, bn=bn_s)), relu=True)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, in_planes: int, planes: int, stride: int = 1) -> None:
        super().__init__()
        self.conv1 = _conv(in_planes, planes, 3, stride)
        self.bn1 = FusedBatchNorm2d(planes)
        self.conv2 = _conv(planes, planes, 3)
        self.bn2 = FusedBatchNorm2d(planes)
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != planes * self.expansion:
            self.shortcut = nn.Sequential(_conv(in_planes, planes * self.expansion, 1, stride),
                                          FusedBatchNorm2d(planes * self.expansion))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        # conv epilogue delivers bn1's batch statistics; xs is x for the shortcut branch -- its gradient is added to conv1's input
        # gradient inside conv1's dgrad epilogue (ops/conv.py) instead of by a separate elementwise kernel
        c1, xs = self.conv1(x, bn=self.bn1, fork=True)
        out = self.bn1(c1, relu=True)
        # bn2 + shortcut add + relu in one pass (ops/norm.py)
        return _bn_residual_relu(self.bn2, self.conv2(out, bn=self.bn2), self.shortcut, xs)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, in_planes: int, planes: int, stride: int = 1) -> None:
        super().__init__()
        self.conv1 = _conv(in_planes, planes, 1)
        self.bn1 = FusedBatchNorm2d(planes)
        self.conv2 = _conv(planes, planes, 3, stride)
        self.bn2 = FusedBatchNorm2d(planes)
        self.conv3 = _conv(planes, planes * self.expansion, 1)
        self.bn3 = FusedBatchNorm2d(planes * self.expansion)
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != planes * self.expansion:
            self.shortcut = nn.Sequential(_conv(in_planes, planes * self.expansion, 1, stride),
                                          FusedBatchNorm2d(planes * self.expansion))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        out = self.bn1(self.conv1(x, bn=self.bn1), relu=True)
        out = self.bn2(self.conv2(out, bn=self.bn2), relu=True)
        return _bn_residual_relu(self.bn3, self.conv3(out, bn=self.bn3), self.shortcut, x)


class ResNet(nn.Module):
    input_shape = (3, 32, 32)

    def __init__(self, block: Type[nn.Module], num_blocks: List[int], num_classes: int = 10, imagenet_stem: bool = False) -> None:
        super().__init__()
        self.num_classes = num_classes
        self.in_planes = 64
        self.imagenet_stem = imagenet_stem
        if imagenet_stem:
            self.input_shape = (3, 224, 224)
            self.conv1 = Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        else:
            self.conv1 = _conv(3, 64, 3)
        self.bn1 = FusedBatchNorm2d(64)
        self.layer1 = self._make_layer(block, 64, num_blocks[0], 1)
        self.layer2 = self._make_layer(block, 128, num_blocks[1], 2)
        self.layer3 = self._make_layer(block, 256, num_blocks[2], 2)
        self.layer4 = self._make_layer(block, 512, num_blocks[3], 2)
        self.linear = Linear(512 * block.expansion, num_classes)

    def _make_layer(self, block, planes: int, n: int, stride: int) -> nn.Sequential:
        layers = []
        for st in [stride] + [1] * (n - 1):
            layers.append(block(self.in_planes, planes, st))
            self.in_planes = planes * block.expansion
        return nn.Sequential(*layers)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        out = self.bn1(self.conv1(x, bn=self.bn1), relu=True)
        if self.imagenet_stem:
            out = F.max_pool2d(out, kernel_size=3, stride=2, padding=1)
        out = self.layer4(self.layer3(self.layer2(self.layer1(out))))
        return self.linear(global_avg_pool(out))          # == F.avg_pool2d(out, 4) on the reference's 4x4 maps

    def name(self) -> str:
        return "resnet"


ResNetSplit = make_split(ResNet, "ResNetSplit")

_CFG = {
    "18": (BasicBlock, [2, 2, 2, 2]),
    "34": (BasicBlock, [3, 4, 6, 3]),
    "50": (Bottleneck, [3, 4, 6, 3]),
    "101": (Bottleneck, [3, 4, 23, 3]),
    "152": (Bottleneck, [3, 8, 36, 3]),
}


def _factory(depth: str, split: bool):
    block, blocks = _CFG[depth]
    cls = ResNetSplit if split else ResNet

    def make(num_classes: int = 10, imagenet_stem: bool = False):
        return cls(block, blocks, num_classes=num_classes, imagenet_stem=imagenet_stem)

    make.__name__ = ("ResNetSplit" if split else "ResNet") + depth
    make.__doc__ = f"ResNet-{depth} (CIFAR variant){' with split-backward drivers' if split else ''}."
    return make


ResNet18, ResNet34, ResNet50, ResNet101, ResNet152 = (_factory(d, False) for d in _CFG)
ResNetSplit18, ResNetSplit34, ResNetSplit50, ResNetSplit101, ResNetSplit152 = (_factory(d, True) for d in _CFG)
