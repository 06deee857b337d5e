"""ResNet-18 / ResNet-50 (BASELINE.json configs 2 and 3), written for channels-last bf16 on H100.

Plain ``torch.nn`` definition (He et al. 2015 topology, torchvision-compatible parameter
names so checkpoints interchange).  Convolutions are library (cuDNN) GEMMs — the framework's own
kernels sit on the parameter-server paths, not here.
"""
from __future__ import annotations

import os
from typing import List, Optional, Type, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.batchnorm import FusedBatchNormAct2d
from ..ops.pooling import FusedMaxPool2d
from ..ops.stem import STEM_K, STEM_STRIDES, stem_conv, stem_conv_fused, stem_fused_supported, stem_supported

# Default (checked by bench/stem_fused_check.py): one implicit-GEMM stem kernel with the BatchNorm
# statistics in its epilogue (csrc/kernels/stem_kernels.cu) instead of im2col + GEMM + statistics pass.
# PSB200_STEM=im2col restores the round-1 path.
_FUSED_STEM = os.environ.get("PSB200_STEM", "fused").lower() != "im2col"
# With the fused stem, BN1 + ReLU + max-pool run as one forward kernel and a two-pass backward that never materialise the
# 112x112 activation or its gradient (ops/batchnorm.py: forward_maxpool); PSB200_STEM_TAIL=unfused keeps the separate kernels.
_FUSED_TAIL = os.environ.get("PSB200_STEM_TAIL", "fused").lower() != "unfused"

def _conv3x3(i, o, stride=1):
    return nn.Conv2d(i, o, 3, stride, 1, bias=False)


def _conv1x1(i, o, stride=1):
    return nn.Conv2d(i, o, 1, stride, 0, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample: Optional[nn.Module] = None):
        super().__init__()
        self.conv1 = _conv3x3(inplanes, planes, stride)
        self.bn1 = FusedBatchNormAct2d(planes, relu=True)          # BN + ReLU in one pass
        self.conv2 = _conv3x3(planes, planes)
        self.bn2 = FusedBatchNormAct2d(planes, relu=True)          # BN + skip add + ReLU in one pass
        self.downsample = downsample

    def forward(self, x):
        identity = x if self.downsample is None else self.downsample(x)
        out = self.bn1(self.conv1(x))
        return self.bn2(self.conv2(out), identity)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample: Optional[nn.Module] = None):
        super().__init__()
        self.conv1 = _conv1x1(inplanes, planes)
        self.bn1 = FusedBatchNormAct2d(planes, relu=True)
        self.conv2 = _conv3x3(planes, planes, stride)
        self.bn2 = FusedBatchNormAct2d(planes, relu=True)
        self.conv3 = _conv1x1(planes, planes * 4)
        self.bn3 = FusedBatchNormAct2d(planes * 4, relu=True)      # BN + skip add + ReLU
        self.downsample = downsample

    def forward(self, x):
        identity = x if self.downsample is None else self.downsample(x)
        out = self.bn1(self.conv1(x))
        out = self.bn2(self.conv2(out))
        return self.bn3(self.conv3(out), identity)


class ResNet(nn.Module):
    def __init__(self, block: Type[Union[BasicBlock, Bottleneck]], layers: List[int],
                 num_classes: int = 1000, zero_init_residual: bool = False, gemm_stem: bool = True):
        super().__init__()
        self.gemm_stem = gemm_stem
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self._engine = None
        self._tag_stem()
        self.bn1 = FusedBatchNormAct2d(64, relu=True)
        self.maxpool = FusedMaxPool2d(3, 2, 1)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], 2)
        self.layer3 = self._make_layer(block, 256, layers[2], 2)
        self.layer4 = self._make_layer(block, 512, layers[3], 2)
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck):
                    nn.init.zeros_(m.bn3.weight)
                elif isinstance(m, BasicBlock):
                    nn.init.zeros_(m.bn2.weight)

    def _tag_stem(self):
        """Ask the PS device engine to keep the stem weight in the zero-padded [64,176] GEMM layout the stem kernel TMA-loads
        (``parallel/layout.py``): the broadcast then delivers it ready for the first forward GEMM."""
        if self.gemm_stem and self.conv1.out_channels == 64:
            self.conv1.weight.ps_arena_layout = (STEM_STRIDES, 64 * STEM_K)

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._tag_stem()                     # conversions may re-create the Parameter object
        return out

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(_conv1x1(self.inplanes, planes * block.expansion, stride),
                                       FusedBatchNormAct2d(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        layers += [block(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def stem(self, x):
        """7x7/2 stem.  An 8-channel input (3 real + 5 zero channels, see ``ops.preprocess``) runs the same
        convolution with the weight zero-padded to 8 input channels: identical math, but the 16-byte pixel
        lets cuDNN use its aligned tensor-core kernels (the 3-channel stem was 23 % of the step)."""
        c = self.conv1
        if x.shape[1] == c.in_channels:
            if self.gemm_stem and stem_supported(x, c):
                return stem_conv(x, c.weight)          # im2col + our wgmma GEMM (C=3 defeats cuDNN)
            return c(x)
        w = F.pad(c.weight, (0, 0, 0, 0, 0, x.shape[1] - c.in_channels))
        if x.is_contiguous(memory_format=torch.channels_last):
            w = w.contiguous(memory_format=torch.channels_last)
        return F.conv2d(x, w, c.bias, c.stride, c.padding, c.dilation, c.groups)

    def _tail(self, y, sums=None):
        """BN1 + ReLU + max-pool after the stem convolution."""
        if sums is not None and _FUSED_TAIL and self.bn1.maxpool_ok(y):
            return self.bn1.forward_maxpool(y, sums)
        return self.maxpool(self.bn1(y, sums=sums) if sums is not None else self.bn1(y))

    def attach(self, optimizer) -> "ResNet":
        """Gate the stem kernel on the parameter server's broadcast: its weight load acquires ``PARAMS_READY`` itself and
        workers stop queueing the separate wait kernel (the stem convolution is the first consumer of parameters in the
        forward pass).  A forward that does not take the fused-stem path falls back to the engine's wait kernel."""
        eng = getattr(optimizer, "_engine", None)
        if eng is None:
            raise ValueError("attach() needs an optimizer running the device engine")
        self._engine = eng
        eng.register_gate(self)
        return self

    def forward(self, x):
        eng = self._engine
        if (_FUSED_STEM and self.gemm_stem and self.training and x.shape[1] == self.conv1.in_channels
                and stem_fused_supported(x, self.conv1)):
            flag_ptr, epoch = eng.gate() if eng is not None else (0, 0)
            y, sums = stem_conv_fused(x, self.conv1.weight, flag_ptr, epoch)   # implicit GEMM + BN statistics in one kernel
            x = self._tail(y, sums)
        else:
            if eng is not None:
                eng.ensure_params()                  # nobody acquired the broadcast in-kernel: the plain wait kernel
            x = self._tail(self.stem(x))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(self.avgpool(x), 1))


def resnet18(num_classes: int = 1000, **kw) -> ResNet:
    return ResNet(BasicBlock, [2, 2, 2, 2], num_classes, **kw)


def resnet50(num_classes: int = 1000, **kw) -> ResNet:
    return ResNet(Bottleneck, [3, 4, 6, 3], num_classes, **kw)
