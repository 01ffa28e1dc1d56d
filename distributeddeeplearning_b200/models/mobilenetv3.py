"""MobileNetV3-Large and -Small (keys, shapes and initialisation match ``torchvision.models.mobilenet_v3_large`` /
``mobilenet_v3_small``).

Every conv + BN + activation is the fused ``conv_bn`` unit: ReLU or hardswish in the BN kernels, the depthwise 3x3 and
5x5 layers on the stencil kernels of csrc/ops/depthwise.cu / depthwise5.cu.  A block is an optional 1x1 expand, a
depthwise k x k, an optional squeeze-excitation (``ops.squeeze_excite``: one autograd node) and a 1x1 linear projection
whose BN adds the block input when the block keeps its shape.  Every width is rounded to a multiple of 8
(``_make_divisible``), SE squeeze widths included, which keeps every layer on the native kernels.
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input
from .mobilenet import _Dropout, _make_divisible

# (input channels, kernel, expanded channels, output channels, SE, activation, stride) as in the MobileNetV3 paper
_LARGE = [(16, 3, 16, 16, False, "RE", 1), (16, 3, 64, 24, False, "RE", 2), (24, 3, 72, 24, False, "RE", 1),
          (24, 5, 72, 40, True, "RE", 2), (40, 5, 120, 40, True, "RE", 1), (40, 5, 120, 40, True, "RE", 1),
          (40, 3, 240, 80, False, "HS", 2), (80, 3, 200, 80, False, "HS", 1), (80, 3, 184, 80, False, "HS", 1),
          (80, 3, 184, 80, False, "HS", 1), (80, 3, 480, 112, True, "HS", 1), (112, 3, 672, 112, True, "HS", 1),
          (112, 5, 672, 160, True, "HS", 2), (160, 5, 960, 160, True, "HS", 1), (160, 5, 960, 160, True, "HS", 1)]
_SMALL = [(16, 3, 16, 16, True, "RE", 2), (16, 3, 72, 24, False, "RE", 2), (24, 3, 88, 24, False, "RE", 1),
          (24, 5, 96, 40, True, "HS", 2), (40, 5, 240, 40, True, "HS", 1), (40, 5, 240, 40, True, "HS", 1),
          (40, 5, 120, 48, True, "HS", 1), (48, 5, 144, 48, True, "HS", 1), (48, 5, 288, 96, True, "HS", 2),
          (96, 5, 576, 96, True, "HS", 1), (96, 5, 576, 96, True, "HS", 1)]


def _bn(c):
    return BatchNorm2d(c, eps=0.001, momentum=0.01)


class ConvBNAct(nn.Sequential):
    """conv + BN + activation (torchvision's ``Conv2dNormActivation``: keys ``.0`` conv, ``.1`` BN); ``act`` is "RE"
    (ReLU), "HS" (hardswish) or None."""

    def __init__(self, cin, cout, kernel_size=3, stride=1, groups=1, act="HS"):
        super().__init__(Conv2d(cin, cout, kernel_size, stride, (kernel_size - 1) // 2, groups=groups), _bn(cout))
        self.act = act

    def forward(self, x, residual=None):
        return conv_bn(x, self[0], self[1], relu=self.act == "RE", residual=residual, hardswish=self.act == "HS")


class SqueezeExcitation(nn.Module):
    """torchvision's ``SqueezeExcitation`` with a hardsigmoid scale: keys ``fc1`` / ``fc2`` (1x1 convs with bias)."""

    def __init__(self, channels, squeeze):
        super().__init__()
        self.fc1 = Conv2d(channels, squeeze, 1, bias=True)
        self.fc2 = Conv2d(squeeze, channels, 1, bias=True)

    def forward(self, x):
        return ops.squeeze_excite(x, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias)


class InvertedResidual(nn.Module):
    def __init__(self, inp, kernel, exp, oup, use_se, act, stride):
        super().__init__()
        if stride not in (1, 2):
            raise ValueError(f"stride should be 1 or 2, got {stride}")
        self.use_res_connect = stride == 1 and inp == oup
        layers = [ConvBNAct(inp, exp, 1, act=act)] if exp != inp else []
        layers.append(ConvBNAct(exp, exp, kernel, stride, groups=exp, act=act))
        if use_se:
            layers.append(SqueezeExcitation(exp, _make_divisible(exp // 4, 8)))
        layers.append(ConvBNAct(exp, oup, 1, act=None))
        self.block = nn.Sequential(*layers)
        self.out_channels = oup

    def forward(self, x):
        h = x
        for m in self.block[:-1]:
            h = m(h)
        # linear bottleneck: no activation; the shortcut is added inside the BN kernel
        return self.block[-1](h, residual=x if self.use_res_connect else None)


class _Hardswish(nn.Module):
    def forward(self, x):
        return ops.hardswish(x)


class MobileNetV3(nn.Module):
    input_size = 224

    def __init__(self, setting, last_channel, num_classes=1000, width_mult=1.0, dropout=0.2):
        super().__init__()
        self.num_classes = num_classes

        def adjust(c):
            return _make_divisible(c * width_mult, 8)

        setting = [(adjust(i), k, adjust(e), adjust(o), se, a, s) for i, k, e, o, se, a, s in setting]
        features = [ConvBNAct(3, setting[0][0], 3, 2, act="HS")]
        features += [InvertedResidual(*cfg) for cfg in setting]
        last_in = setting[-1][3]
        features.append(ConvBNAct(last_in, 6 * last_in, 1, act="HS"))
        self.features = nn.Sequential(*features)
        self.last_channel = adjust(last_channel)
        self.classifier = nn.Sequential(Linear(6 * last_in, self.last_channel), _Hardswish(), _Dropout(dropout),
                                        Linear(self.last_channel, num_classes))
        for m in self.modules():
            if isinstance(m, Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
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
        if x.shape[1] != self.last_channel:        # the native GEMM's padded width
            x = x[:, : self.last_channel].contiguous()
        x = self.classifier[1](x)
        x = self.classifier[2](x)
        return self.classifier[3](x)[:, : self.num_classes]


def mobilenet_v3_large(num_classes=1000, width_mult=1.0, **kw):
    return MobileNetV3(_LARGE, 1280, num_classes=num_classes, width_mult=width_mult, **kw)


def mobilenet_v3_small(num_classes=1000, width_mult=1.0, **kw):
    return MobileNetV3(_SMALL, 1024, num_classes=num_classes, width_mult=width_mult, **kw)
