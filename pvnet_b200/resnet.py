"""Dilated ResNet-18 trunk with the reference's parameter names.

Mirrors what zju3dv/pvnet's ``lib/networks/resnet.py`` builds for
``resnet18(fully_conv=True, output_stride=8, remove_avg_pool_layer=True)``
(reference :120-220): stages whose stride would push the output stride past 8 keep
stride 1 and dilate instead (:173-183), and *every* block of such a stage, including
its first, uses the new dilation (:193-196).  ``forward`` returns the six feature
maps the reference returns (:220).  Module/parameter names match the reference so its
checkpoints load with ``load_state_dict`` (SURVEY.md §8b "Weights").

This PyTorch graph is what train mode (BatchNorm batch statistics, autograd) runs;
eval-mode inference goes through the native sm_90a path in
``pvnet_b200.model_repository.Resnet18_8s``.
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


class DilatedResNet18(nn.Module):
    """conv1/bn1/maxpool + layer1..4 (2 BasicBlocks each) + a caller-supplied `fc` head."""

    def __init__(self, output_stride=8):
        super().__init__()
        self.output_stride = output_stride
        self._stride_so_far = 4
        self._dilation = 1
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, stride=2, padding=1)
        self.layer1 = self._stage(64, 2, stride=1)
        self.layer2 = self._stage(128, 2, stride=2)
        self.layer3 = self._stage(256, 2, stride=2)
        self.layer4 = self._stage(512, 2, stride=2)
        self.fc = nn.Identity()          # replaced by Resnet18_8s (model_repository.py:22-26 in the reference)
        for mod in self.modules():       # reference init, :162-168
            if isinstance(mod, nn.Conv2d):
                n = mod.kernel_size[0] * mod.kernel_size[1] * mod.out_channels
                mod.weight.data.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(mod, nn.BatchNorm2d):
                mod.weight.data.fill_(1)
                mod.bias.data.zero_()

    def _stage(self, planes, blocks, stride):
        down = None
        if stride != 1 or self.inplanes != planes:
            if self._stride_so_far == self.output_stride:
                self._dilation *= stride          # keep resolution, dilate instead
                stride = 1
            else:
                self._stride_so_far *= stride
            down = nn.Sequential(nn.Conv2d(self.inplanes, planes, 1, stride=stride, bias=False),
                                 nn.BatchNorm2d(planes))
        layers = [BasicBlock(self.inplanes, planes, stride, down, dilation=self._dilation)]
        self.inplanes = planes
        layers += [BasicBlock(planes, planes, dilation=self._dilation) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x2s = self.relu(self.bn1(self.conv1(x)))
        x4s = self.layer1(self.maxpool(x2s))
        x8s = self.layer2(x4s)
        x16s = self.layer3(x8s)
        x32s = self.layer4(x16s)
        return x2s, x4s, x8s, x16s, x32s, self.fc(x32s)


def resnet18(output_stride=8, **_ignored):
    """The reference's `resnet18(fully_conv=True, pretrained=True, output_stride=8,
    remove_avg_pool_layer=True)` minus the ImageNet download (reference :231 fetches
    weights over the network; there is none here -- load a checkpoint instead)."""
    return DilatedResNet18(output_stride=output_stride)
