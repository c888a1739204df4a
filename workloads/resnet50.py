"""ResNet-50 (He et al. 2015, v1.5 stride placement as in torchvision) in plain torch.nn — the model
BASELINE.json config 2 names.  25,557,032 parameters, 161 parameter tensors; random init (no
network for checkpoints).

Every batch norm is applied through torch_on_k8s_b200.fused_bn together with the ReLU and residual
add that follow it: on CUDA bf16 channels_last training inputs that is one fused libtok8s kernel
per site, bit-identical to the unfused ops; anything else runs the plain nn composition.  The stem's
max pool runs through fused_bn.max_pool under the same conditions.

A block hands its output to the next block as a pair (x, x_short), one for conv1 and one for the
shortcut, so that the fused backward receives the two gradients separately and sums them inside its
reduction instead of after an autograd add (fused_bn.bn_add_relu's `shortcut`).  The last block
returns its output alone to the average pool."""
from __future__ import annotations

import torch
import torch.nn as nn

from torch_on_k8s_b200.fused_bn import bn2_add_relu, bn_add_relu, bn_relu, max_pool


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes: int, planes: int, stride: int = 1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * self.expansion, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.fork = True  # return (y, y) for the next block's conv1 and shortcut

    def forward(self, x):
        x, x_short = x if isinstance(x, tuple) else (x, x)
        out = bn_relu(self.conv1(x), self.bn1)
        out = bn_relu(self.conv2(out), self.bn2)
        out = self.conv3(out)
        if self.downsample is not None:
            # downsample = Sequential(conv, bn): its batch norm is fused into the residual add
            conv_d, bn_d = self.downsample
            return bn2_add_relu(out, self.bn3, conv_d(x_short), bn_d, shortcut=self.fork)
        return bn_add_relu(out, self.bn3, x_short, shortcut=self.fork)


class ResNet50(nn.Module):
    def __init__(self, num_classes: int = 1000):
        super().__init__()
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, stride=2, padding=1)
        self.layer1 = self._make_layer(64, 3, 1)
        self.layer2 = self._make_layer(128, 4, 2)
        self.layer3 = self._make_layer(256, 6, 2)
        self.layer4 = self._make_layer(512, 3, 2)
        self.layer4[-1].fork = False
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512 * Bottleneck.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def _make_layer(self, planes: int, blocks: int, stride: int):
        downsample = None
        if stride != 1 or self.inplanes != planes * Bottleneck.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * Bottleneck.expansion, 1, stride=stride, bias=False),
                nn.BatchNorm2d(planes * Bottleneck.expansion))
        layers = [Bottleneck(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * Bottleneck.expansion
        for _ in range(1, blocks):
            layers.append(Bottleneck(self.inplanes, planes))
        return nn.Sequential(*layers)

    def forward(self, x):
        x = max_pool(bn_relu(self.conv1(x), self.bn1), self.maxpool)
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        x = torch.flatten(self.avgpool(x), 1)
        return self.fc(x)


def resnet50(num_classes: int = 1000) -> ResNet50:
    return ResNet50(num_classes)
