"""ResNet family used by the reference's benchmarks (reference README.md:20-22,
run_deepreduce.sh:11,20,33): CIFAR ResNet-20 (269 722 params incl. fc, paper
Table 1) and ImageNet ResNet-50 (25 557 032 params).  Plain ``torch.nn``;
convolutions run on cuDNN (library GEMM/conv is the model compute, the
framework's own kernels are the gradient exchange).
"""
from __future__ import annotations

import torch.nn as nn
import torch.nn.functional as F

from .fused_bn import bn_add_relu, bn_bn_add_relu, bn_relu, bn_relu_maxpool


# ----------------------------------------------------------------------------
# CIFAR ResNet (He et al. 2015, 6n+2 layers): resnet20 = n 3
# ----------------------------------------------------------------------------
class _BasicCifar(nn.Module):
    def __init__(self, inp, out, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(inp, out, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(out)
        self.conv2 = nn.Conv2d(out, out, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(out)
        self.pad = None
        if stride != 1 or inp != out:
            self.pad = (out - inp, stride)        # option A: strided identity + zero channel padding

    def forward(self, x):
        y = F.relu(self.bn1(self.conv1(x)))
        y = self.bn2(self.conv2(y))
        if self.pad is not None:
            extra, s = self.pad
            x = F.pad(x[:, :, ::s, ::s], (0, 0, 0, 0, extra // 2, extra - extra // 2))
        return F.relu(x + y)


class ResNetCifar(nn.Module):
    def __init__(self, n: int = 3, num_classes: int = 10):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 16, 3, 1, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(16)
        layers, inp = [], 16
        for out, stride in ((16, 1), (32, 2), (64, 2)):
            for i in range(n):
                layers.append(_BasicCifar(inp, out, stride if i == 0 else 1))
                inp = out
        self.layers = nn.Sequential(*layers)
        self.fc = nn.Linear(64, num_classes)

    def forward(self, x):
        x = F.relu(self.bn1(self.conv1(x)))
        x = self.layers(x)
        x = F.adaptive_avg_pool2d(x, 1).flatten(1)
        return self.fc(x)


def resnet20(num_classes: int = 10) -> ResNetCifar:
    return ResNetCifar(3, num_classes)


# ----------------------------------------------------------------------------
# ImageNet ResNet-50 (v1.5: stride on the 3x3)
# ----------------------------------------------------------------------------
class _Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inp, width, stride, downsample):
        super().__init__()
        out = width * self.expansion
        self.conv1 = nn.Conv2d(inp, width, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = nn.Conv2d(width, width, 3, stride, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = nn.Conv2d(width, out, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(out)
        self.downsample = None
        if downsample:
            self.downsample = nn.Sequential(nn.Conv2d(inp, out, 1, stride, bias=False), nn.BatchNorm2d(out))

    def forward(self, x, skip=None, fork=False):
        # each helper is the unfused composite unless its input is a channels_last bf16 CUDA training tensor
        # (models/fused_bn.py); either way the results are bitwise the same.  skip: the block input as the skip path
        # reads it, when the producer returned it as a second output.  fork: return (output for the next conv1, output
        # for the next skip path or None), so backward gets the two gradients apart.  Only the identity tail forks;
        # for the downsample tail the second gradient did not pay (DESIGN.md §8a), and it returns (output, None).
        skip = x if skip is None else skip
        xd = None if self.downsample is None else self.downsample[0](skip)
        y = bn_relu(self.conv1(x), self.bn1)
        y = bn_relu(self.conv2(y), self.bn2)
        y = self.conv3(y)
        if xd is None:
            return bn_add_relu(y, self.bn3, skip, fork=fork)
        o = bn_bn_add_relu(y, self.bn3, xd, self.downsample[1])
        return (o, None) if fork else o


class ResNet(nn.Module):
    def __init__(self, blocks=(3, 4, 6, 3), num_classes: int = 1000):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        stages, inp = [], 64
        for i, (n, width) in enumerate(zip(blocks, (64, 128, 256, 512))):
            for j in range(n):
                stride = 2 if (j == 0 and i > 0) else 1
                stages.append(_Bottleneck(inp, width, stride, downsample=(j == 0)))
                inp = width * 4
        self.layers = nn.Sequential(*stages)
        self.fc = nn.Linear(inp, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def forward(self, x):
        # every block input feeds conv1 and the skip path; an identity tail returns it once per consumer (fork), so
        # its backward adds the two gradients itself.  The stem stays on one output (DESIGN.md §8a).
        x, skip = bn_relu_maxpool(self.conv1(x), self.bn1, self.maxpool), None
        for blk in self.layers:
            x, skip = blk(x, skip, fork=True)
        x = F.adaptive_avg_pool2d(x, 1).flatten(1)
        return self.fc(x)


def resnet50(num_classes: int = 1000) -> ResNet:
    return ResNet((3, 4, 6, 3), num_classes)
