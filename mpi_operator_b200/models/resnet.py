"""ResNet v1.5 family (He et al.) for synthetic-ImageNet throughput runs.

This is the architecture tf_cnn_benchmarks trains for ``--model=resnet101``
in the reference's headline example (examples/v2beta1/tensorflow-benchmarks/
tensorflow-benchmarks.yaml:38-42, README.md:180-212): bottleneck blocks
[3, 4, 23, 3], 44.5 M parameters, 224x224x3 inputs, 1000 classes.
"""
from __future__ import annotations

from typing import List, Type

import torch
import torch.nn as nn

from ..ops.fused_bn import ResidualLink, bn_act, conv_bn_act


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        idt = x if self.downsample is None else self.downsample(x)
        out = bn_act(self.bn1, self.conv1(x))
        return bn_act(self.bn2, self.conv2(out), residual=idt)  # fused BN + add + ReLU


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        # v1.5: the stride sits on the 3x3 conv
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x):
        idt = x if self.downsample is None else self.downsample(x)
        # residual == conv1's input: conv3's backward can hand the residual gradient to conv1's dgrad (ops/fused_bn.py)
        link = ResidualLink() if self.downsample is None else None
        out = conv_bn_act(self.conv1, self.bn1, x, link=link)   # 1x1: BN statistics can come from the GEMM epilogue
        out = bn_act(self.bn2, self.conv2(out))
        return conv_bn_act(self.conv3, self.bn3, out, residual=idt, link=link)  # 1x1 + fused BN + add + ReLU


class _Downsample(nn.Sequential):
    """1x1 conv + BN on the shortcut (same parameter names as nn.Sequential(conv, bn): '0', '1')."""

    def __init__(self, inplanes: int, outplanes: int, stride: int):
        super().__init__(nn.Conv2d(inplanes, outplanes, 1, stride, bias=False), nn.BatchNorm2d(outplanes))

    def forward(self, x):
        return bn_act(self[1], self[0](x), relu=False)


class ResNet(nn.Module):
    def __init__(self, block: Type[nn.Module], layers: List[int], num_classes: int = 1000, width: int = 64):
        super().__init__()
        self.inplanes = width
        self.conv1 = nn.Conv2d(3, width, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        self.layer1 = self._make(block, width, layers[0], 1)
        self.layer2 = self._make(block, width * 2, layers[1], 2)
        self.layer3 = self._make(block, width * 4, layers[2], 2)
        self.layer4 = self._make(block, width * 8, layers[3], 2)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(width * 8 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        for m in self.modules():  # zero-init the last BN of each residual branch
            if isinstance(m, Bottleneck):
                nn.init.zeros_(m.bn3.weight)
            elif isinstance(m, BasicBlock):
                nn.init.zeros_(m.bn2.weight)

    def _make(self, block, planes, blocks, stride):
        down = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            down = _Downsample(self.inplanes, planes * block.expansion, stride)
        layers = [block(self.inplanes, planes, stride, down)]
        self.inplanes = planes * block.expansion
        layers += [block(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.maxpool(bn_act(self.bn1, self.conv1(x)))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(self.avgpool(x), 1))


def resnet18(**kw): return ResNet(BasicBlock, [2, 2, 2, 2], **kw)  # noqa: E704
def resnet50(**kw): return ResNet(Bottleneck, [3, 4, 6, 3], **kw)  # noqa: E704
def resnet101(**kw): return ResNet(Bottleneck, [3, 4, 23, 3], **kw)  # noqa: E704
def resnet152(**kw): return ResNet(Bottleneck, [3, 8, 36, 3], **kw)  # noqa: E704
