"""DenseNet-121/161/169/201 (keys match ``torchvision.models.densenet*``).

The reference's benchmark resolves ``--model`` against every torchvision constructor
(``PyTorch_benchmark/src/pytorch_synthetic_benchmark.py:60``), which includes the DenseNet family of torchvision
0.2.1 (SURVEY.md 2.7).  A dense layer is pre-activation — ``norm1 -> relu -> conv1(1x1) -> norm2 -> relu ->
conv2(3x3)`` — so it maps onto: one standalone BN+ReLU kernel (``ops.batch_norm_act``), one fused conv+BN+ReLU unit
and one plain conv; the growing feature map is assembled by the native channel-concat kernel.  All widths are
multiples of 16, which the wgmma conv kernels accept (partial 64-channel k-blocks are zero-filled by TMA).
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, bn_act, conv_bn, conv_bn_pool, prepare_input


class _DenseLayer(nn.Module):
    def __init__(self, cin, growth, bn_size):
        super().__init__()
        self.norm1 = BatchNorm2d(cin)
        self.conv1 = Conv2d(cin, bn_size * growth, 1)
        self.norm2 = BatchNorm2d(bn_size * growth)
        self.conv2 = Conv2d(bn_size * growth, growth, 3, padding=1)

    def forward(self, x):
        h = bn_act(x, self.norm1, relu=True)
        h = conv_bn(h, self.conv1, self.norm2, relu=True)
        return self.conv2(h)


class _DenseBlock(nn.Module):
    def __init__(self, layers, cin, growth, bn_size):
        super().__init__()
        for i in range(layers):
            self.add_module(f"denselayer{i + 1}", _DenseLayer(cin + i * growth, growth, bn_size))

    def forward(self, x):
        feats = x
        for layer in self.children():
            feats = ops.concat_channels([feats, layer(feats)])
        return feats


class _Transition(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.norm = BatchNorm2d(cin)
        self.conv = Conv2d(cin, cout, 1)

    def forward(self, x):
        return ops.avg_pool2d(self.conv(bn_act(x, self.norm, relu=True)), 2, 2)


class _Features(nn.Module):
    def __init__(self, growth, block_config, init_features, bn_size):
        super().__init__()
        self.conv0 = Conv2d(3, init_features, 7, stride=2, padding=3)
        self.norm0 = BatchNorm2d(init_features)
        c = init_features
        for i, n in enumerate(block_config):
            self.add_module(f"denseblock{i + 1}", _DenseBlock(n, c, growth, bn_size))
            c += n * growth
            if i != len(block_config) - 1:
                self.add_module(f"transition{i + 1}", _Transition(c, c // 2))
                c //= 2
        self.norm5 = BatchNorm2d(c)
        self.out_channels = c

    def forward(self, x):
        x = conv_bn_pool(x, self.conv0, self.norm0, 3, 2, 1)
        for name, m in self.named_children():
            if name.startswith(("denseblock", "transition")):
                x = m(x)
        return bn_act(x, self.norm5, relu=True)


class DenseNet(nn.Module):
    input_size = 224

    def __init__(self, growth_rate=32, block_config=(6, 12, 24, 16), num_init_features=64, bn_size=4, num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.features = _Features(growth_rate, block_config, num_init_features, bn_size)
        self.classifier = Linear(self.features.out_channels, num_classes)
        for m in self.modules():
            if isinstance(m, Conv2d):
                nn.init.kaiming_normal_(m.weight)
            elif isinstance(m, Linear):
                nn.init.zeros_(m.bias)

    def forward(self, x):
        x = self.features(prepare_input(x))
        x = ops.global_avg_pool(x)
        return self.classifier(x)


def densenet121(**kw):
    return DenseNet(32, (6, 12, 24, 16), 64, **kw)


def densenet169(**kw):
    return DenseNet(32, (6, 12, 32, 32), 64, **kw)


def densenet201(**kw):
    return DenseNet(32, (6, 12, 48, 32), 64, **kw)


def densenet161(**kw):
    return DenseNet(48, (6, 12, 36, 24), 96, **kw)
