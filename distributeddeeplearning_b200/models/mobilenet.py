"""MobileNetV2 (keys, shapes and initialisation match ``torchvision.models.mobilenet_v2``).

Every layer is conv + BN + activation through the fused ``conv_bn`` unit.  An inverted-residual block is a 1x1 expand
(ReLU6), a depthwise 3x3 (ReLU6; the stencil kernels of csrc/ops/depthwise.cu) and a 1x1 linear projection whose BN
adds the block input when the block keeps its shape.  torchvision's ``_make_divisible`` rounds every width to a multiple
of 8, which also keeps every layer on the native kernels.
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input


def _make_divisible(v: float, divisor: int, min_value=None) -> int:
    """torchvision's channel rounding: the nearest multiple of ``divisor`` that is not below 90 % of ``v``."""
    if min_value is None:
        min_value = divisor
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


class ConvBNReLU6(nn.Sequential):
    """conv + BN + ReLU6 (torchvision's ``Conv2dNormActivation``: keys ``.0`` conv, ``.1`` BN)."""

    def __init__(self, cin, cout, kernel_size=3, stride=1, groups=1):
        super().__init__(Conv2d(cin, cout, kernel_size, stride, (kernel_size - 1) // 2, groups=groups), BatchNorm2d(cout))

    def forward(self, x):
        return conv_bn(x, self[0], self[1], relu6=True)


class InvertedResidual(nn.Module):
    def __init__(self, inp, oup, stride, expand_ratio):
        super().__init__()
        if stride not in (1, 2):
            raise ValueError(f"stride should be 1 or 2, got {stride}")
        hidden = int(round(inp * expand_ratio))
        self.use_res_connect = stride == 1 and inp == oup
        layers = [ConvBNReLU6(inp, hidden, 1)] if expand_ratio != 1 else []
        layers += [ConvBNReLU6(hidden, hidden, 3, stride, groups=hidden), Conv2d(hidden, oup, 1), BatchNorm2d(oup)]
        self.conv = nn.Sequential(*layers)
        self.out_channels = oup

    def forward(self, x):
        h = x
        for m in self.conv[:-2]:
            h = m(h)
        # linear bottleneck: no activation; the shortcut is added inside the BN kernel
        return conv_bn(h, self.conv[-2], self.conv[-1], relu=False, residual=x if self.use_res_connect else None)


class _Dropout(nn.Module):
    def __init__(self, p):
        super().__init__()
        self.p = p

    def forward(self, x):
        return ops.dropout(x, self.p, self.training)


class MobileNetV2(nn.Module):
    input_size = 224

    def __init__(self, num_classes=1000, width_mult=1.0, round_nearest=8, dropout=0.2):
        super().__init__()
        self.num_classes = num_classes
        setting = [[1, 16, 1, 1], [6, 24, 2, 2], [6, 32, 3, 2], [6, 64, 4, 2], [6, 96, 3, 1], [6, 160, 3, 2],
                   [6, 320, 1, 1]]       # expansion t, output channels c, repeats n, first stride s
        inp = _make_divisible(32 * width_mult, round_nearest)
        self.last_channel = _make_divisible(1280 * max(1.0, width_mult), round_nearest)
        features = [ConvBNReLU6(3, inp, stride=2)]
        for t, c, n, s in setting:
            oup = _make_divisible(c * width_mult, round_nearest)
            for i in range(n):
                features.append(InvertedResidual(inp, oup, s if i == 0 else 1, t))
                inp = oup
        features.append(ConvBNReLU6(inp, self.last_channel, 1))
        self.features = nn.Sequential(*features)
        self.classifier = nn.Sequential(_Dropout(dropout), Linear(self.last_channel, num_classes))
        for m in self.modules():
            if isinstance(m, Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
            elif isinstance(m, BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
            elif isinstance(m, Linear):
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.zeros_(m.bias)

    def forward(self, x):
        x = prepare_input(x)
        x = self.features(x)
        x = ops.global_avg_pool(x)
        x = self.classifier[0](x)
        return self.classifier[1](x)[:, : self.num_classes]


def mobilenet_v2(num_classes=1000, width_mult=1.0, **kw):
    return MobileNetV2(num_classes=num_classes, width_mult=width_mult, **kw)
