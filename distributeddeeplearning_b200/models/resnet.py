"""ResNet-18/34/50/101/152 (v1.5: stride on the 3x3 of each bottleneck).

Architecture and state_dict keys match ``torchvision.models.resnet*`` — the models the reference
instantiates by name (``PyTorch_benchmark/src/pytorch_synthetic_benchmark.py:60``,
``PyTorch_imagenet/src/imagenet_pytorch_horovod.py:383``, ``PyTorch_hvd/...:115``; the TF twin
builds the same v1.5 variant, ``TensorFlow_imagenet/src/resnet_model.py:193-195,237-320``).
Every conv+BN(+ReLU)(+residual) is ONE fused op (``ops.conv_bn_act``): wgmma implicit GEMM with
BN statistics in its epilogue, then a single BN-apply/ReLU/add pass.
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from ..ops.blocks import residual_block, residual_block_supported
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input, conv_bn_pool


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = Conv2d(inplanes, planes, 3, stride, 1)
        self.bn1 = BatchNorm2d(planes)
        self.conv2 = Conv2d(planes, planes, 3, 1, 1)
        self.bn2 = BatchNorm2d(planes)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        convs, bns = (self.conv1, self.conv2), (self.bn1, self.bn2)
        if residual_block_supported(x, convs, bns, self.downsample):
            return residual_block(x, convs, bns, self.downsample)      # one autograd node, fused input-grad sum
        identity = x
        out = conv_bn(x, self.conv1, self.bn1, relu=True)
        if self.downsample is not None:
            identity = conv_bn(x, self.downsample[0], self.downsample[1], relu=False)
        return conv_bn(out, self.conv2, self.bn2, relu=True, residual=identity)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = Conv2d(inplanes, planes, 1)
        self.bn1 = BatchNorm2d(planes)
        self.conv2 = Conv2d(planes, planes, 3, stride, 1)
        self.bn2 = BatchNorm2d(planes)
        self.conv3 = Conv2d(planes, planes * 4, 1)
        self.bn3 = BatchNorm2d(planes * 4)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        convs, bns = (self.conv1, self.conv2, self.conv3), (self.bn1, self.bn2, self.bn3)
        if residual_block_supported(x, convs, bns, self.downsample):
            return residual_block(x, convs, bns, self.downsample)      # one autograd node, fused input-grad sum
        identity = x
        out = conv_bn(x, self.conv1, self.bn1, relu=True)
        out = conv_bn(out, self.conv2, self.bn2, relu=True)
        if self.downsample is not None:
            identity = conv_bn(x, self.downsample[0], self.downsample[1], relu=False)
        return conv_bn(out, self.conv3, self.bn3, relu=True, residual=identity)


class ResNet(nn.Module):
    input_size = 224

    def __init__(self, block, layers, num_classes=1000, zero_init_residual=False):
        super().__init__()
        self.num_classes = num_classes
        self.inplanes = 64
        self.conv1 = Conv2d(3, 64, 7, 2, 3)
        self.bn1 = BatchNorm2d(64)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=2)
        self.fc = Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck):
                    nn.init.zeros_(m.bn3.weight)
                elif isinstance(m, BasicBlock):
                    nn.init.zeros_(m.bn2.weight)

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(Conv2d(self.inplanes, planes * block.expansion, 1, stride),
                                       BatchNorm2d(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes))
        return nn.Sequential(*layers)

    def forward(self, x):
        x = prepare_input(x)
        x = conv_bn_pool(x, self.conv1, self.bn1, 3, 2, 1)      # conv1 + bn1 + relu + maxpool as one unit
        x = self.layer1(x)
        x = self.layer2(x)
        x = self.layer3(x)
        x = self.layer4(x)
        x = ops.global_avg_pool(x)
        return self.fc(x)[:, : self.num_classes]


def resnet18(**kw):
    return ResNet(BasicBlock, [2, 2, 2, 2], **kw)


def resnet34(**kw):
    return ResNet(BasicBlock, [3, 4, 6, 3], **kw)


def resnet50(**kw):
    return ResNet(Bottleneck, [3, 4, 6, 3], **kw)


def resnet101(**kw):
    return ResNet(Bottleneck, [3, 4, 23, 3], **kw)


def resnet152(**kw):
    return ResNet(Bottleneck, [3, 8, 36, 3], **kw)
