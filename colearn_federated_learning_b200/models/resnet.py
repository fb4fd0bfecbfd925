"""ResNet-18 (BASELINE config 4: bf16 on synthetic 32x32 images, 10 classes).

Not present in the reference (SURVEY §2.5 K17).  Structure and state-dict keys follow the
canonical ImageNet ResNet-18 (7x7 stem, max-pool, 4 stages of 2 BasicBlocks, global avg-pool,
fc) so that with ``num_classes=10`` the parameter count is the 11 181 642 (+9 620 BN buffers)
quoted in SURVEY §2.5.  This module is the architecture + state-dict definition (and the CPU /
eval path); local training on a GPU runs through ``fl/convnet.py`` — im2col + wgmma GEMMs +
this repo's BatchNorm / pooling kernels — and the federated part (flat-arena broadcast, FedAvg
reduce/apply, SGD, loss) through the comm / elementwise kernels.  BN running statistics are
buffers and are *not* averaged by default, which is the reference FedAvg semantics (parameters
only, SURVEY §2.3); ``average_buffers=True`` on the engine opts in.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes: int, planes: int, stride: int = 1) -> None:
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.downsample = None
        if stride != 1 or inplanes != planes:
            self.downsample = nn.Sequential(
                nn.Conv2d(inplanes, planes, 1, stride, bias=False), nn.BatchNorm2d(planes))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        identity = x if self.downsample is None else self.downsample(x)
        out = F.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        return F.relu(out + identity)


class ResNet18(nn.Module):
    def __init__(self, num_classes: int = 10) -> None:
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.layer1 = nn.Sequential(BasicBlock(64, 64), BasicBlock(64, 64))
        self.layer2 = nn.Sequential(BasicBlock(64, 128, 2), BasicBlock(128, 128))
        self.layer3 = nn.Sequential(BasicBlock(128, 256, 2), BasicBlock(256, 256))
        self.layer4 = nn.Sequential(BasicBlock(256, 512, 2), BasicBlock(512, 512))
        self.fc = nn.Linear(512, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = F.relu(self.bn1(self.conv1(x)))
        x = F.max_pool2d(x, 3, 2, 1)
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        x = torch.flatten(F.adaptive_avg_pool2d(x, 1), 1)
        return self.fc(x)
