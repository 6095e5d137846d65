"""Dilated ResNet-18 / 34 / 50 trunks with the reference's parameter names.

Mirrors what zju3dv/pvnet's ``lib/networks/resnet.py`` builds for
``resnet18/34/50(fully_conv=True, output_stride=8, remove_avg_pool_layer=True)``
(reference :73-220): stages whose stride would push the output stride past 8 keep
stride 1 and dilate instead (:173-183), and *every* block of such a stage, including
its first, uses the new dilation (:193-196); the 1x1 downsample is never dilated.  In a
Bottleneck the stride and the dilation sit on conv2, the 3x3 (:73-91).  ``forward``
returns the six feature maps the reference returns (:220).  Module/parameter names match
the reference so its checkpoints load with ``load_state_dict`` (SURVEY.md §8b "Weights").

This PyTorch graph is what train mode (BatchNorm batch statistics, autograd) runs;
eval-mode inference goes through the native sm_90a path in
``pvnet_b200.model_repository``.
"""
from __future__ import annotations

import math

import torch.nn as nn


def conv3x3(cin, cout, stride=1, dilation=1):
    # "full" padding for a dilated 3x3 kernel == dilation (reference :22-37)
    return nn.Conv2d(cin, cout, 3, stride=stride, padding=dilation, dilation=dilation, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, cin, cout, stride=1, downsample=None, dilation=1):
        super().__init__()
        self.conv1 = conv3x3(cin, cout, stride, dilation)
        self.bn1 = nn.BatchNorm2d(cout)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = conv3x3(cout, cout, 1, dilation)
        self.bn2 = nn.BatchNorm2d(cout)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        y = self.relu(self.bn1(self.conv1(x)))
        y = self.bn2(self.conv2(y))
        skip = x if self.downsample is None else self.downsample(x)
        return self.relu(y + skip)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, cin, planes, stride=1, downsample=None, dilation=1):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = conv3x3(planes, planes, stride, dilation)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        y = self.relu(self.bn1(self.conv1(x)))
        y = self.relu(self.bn2(self.conv2(y)))
        y = self.bn3(self.conv3(y))
        skip = x if self.downsample is None else self.downsample(x)
        return self.relu(y + skip)


class DilatedResNet(nn.Module):
    """conv1/bn1/maxpool + layer1..4 (`blocks[i]` blocks of `block` each) + a caller-supplied `fc` head."""

    def __init__(self, block, blocks, output_stride=8):
        super().__init__()
        self.output_stride = output_stride
        self._stride_so_far = 4
        self._dilation = 1
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, stride=2, padding=1)
        self.layer1 = self._stage(block, 64, blocks[0], stride=1)
        self.layer2 = self._stage(block, 128, blocks[1], stride=2)
        self.layer3 = self._stage(block, 256, blocks[2], stride=2)
        self.layer4 = self._stage(block, 512, blocks[3], stride=2)
        self.fc = nn.Identity()          # replaced by Resnet*_8s (model_repository.py:22-26 in the reference)
        for mod in self.modules():       # reference init, :162-168
            if isinstance(mod, nn.Conv2d):
                n = mod.kernel_size[0] * mod.kernel_size[1] * mod.out_channels
                mod.weight.data.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(mod, nn.BatchNorm2d):
                mod.weight.data.fill_(1)
                mod.bias.data.zero_()

    def _stage(self, block, planes, blocks, stride):
        down = None
        cout = planes * block.expansion
        if stride != 1 or self.inplanes != cout:
            if self._stride_so_far == self.output_stride:
                self._dilation *= stride          # keep resolution, dilate instead
                stride = 1
            else:
                self._stride_so_far *= stride
            down = nn.Sequential(nn.Conv2d(self.inplanes, cout, 1, stride=stride, bias=False), nn.BatchNorm2d(cout))
        layers = [block(self.inplanes, planes, stride, down, dilation=self._dilation)]
        self.inplanes = cout
        layers += [block(cout, planes, dilation=self._dilation) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x2s = self.relu(self.bn1(self.conv1(x)))
        x4s = self.layer1(self.maxpool(x2s))
        x8s = self.layer2(x4s)
        x16s = self.layer3(x8s)
        x32s = self.layer4(x16s)
        return x2s, x4s, x8s, x16s, x32s, self.fc(x32s)


class DilatedResNet18(DilatedResNet):
    """conv1/bn1/maxpool + layer1..4 (2 BasicBlocks each) + a caller-supplied `fc` head."""

    def __init__(self, output_stride=8):
        super().__init__(BasicBlock, (2, 2, 2, 2), output_stride)


# The reference's constructors minus the ImageNet download (reference :230-255 fetch weights over the network;
# there is none here -- load a checkpoint instead).
def resnet18(output_stride=8, **_ignored):
    """`resnet18(fully_conv=True, pretrained=True, output_stride=8, remove_avg_pool_layer=True)`: 2-2-2-2 BasicBlocks."""
    return DilatedResNet18(output_stride=output_stride)


def resnet34(output_stride=8, **_ignored):
    """`resnet34(...)` as Resnet34_8s builds it: 3-4-6-3 BasicBlocks."""
    return DilatedResNet(BasicBlock, (3, 4, 6, 3), output_stride)


def resnet50(output_stride=8, **_ignored):
    """`resnet50(...)` as Resnet50_8s builds it: 3-4-6-3 Bottlenecks (expansion 4)."""
    return DilatedResNet(Bottleneck, (3, 4, 6, 3), output_stride)
