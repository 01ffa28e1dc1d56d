"""EfficientNet-B0 to -B7 (keys, shapes and initialisation match ``torchvision.models.efficientnet_b0`` ...
``efficientnet_b7``).

Every conv + BN + activation is the fused ``conv_bn`` unit with SiLU in the BN kernels; the depthwise 3x3 and 5x5 layers
run on the stencil kernels of csrc/ops/depthwise.cu / depthwise5.cu.  An MBConv block is an optional 1x1 expand, a
depthwise k x k, a squeeze-excitation with a SiLU inner activation and a sigmoid gate (``ops.squeeze_excite``, one
autograd node, any squeeze width) and a 1x1 linear projection.  When the block keeps its shape, the projection's BN
also applies stochastic depth (one keep scale per sample, drawn on the device) and adds the block input, in one kernel.
"""
from __future__ import annotations

import math

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input
from .mobilenet import _Dropout, _make_divisible

# (expand ratio, kernel, stride, input channels, output channels, layers) of the seven stages, before width / depth scaling
_STAGES = [(1, 3, 1, 32, 16, 1), (6, 3, 2, 16, 24, 2), (6, 5, 2, 24, 40, 2), (6, 3, 2, 40, 80, 3),
           (6, 5, 1, 80, 112, 3), (6, 5, 2, 112, 192, 4), (6, 3, 1, 192, 320, 1)]
# variant -> (width multiplier, depth multiplier, classifier dropout, crop size) as in torchvision 0.26
_VARIANTS = {"efficientnet_b0": (1.0, 1.0, 0.2, 224), "efficientnet_b1": (1.0, 1.1, 0.2, 240),
             "efficientnet_b2": (1.1, 1.2, 0.3, 288), "efficientnet_b3": (1.2, 1.4, 0.3, 300),
             "efficientnet_b4": (1.4, 1.8, 0.4, 380), "efficientnet_b5": (1.6, 2.2, 0.4, 456),
             "efficientnet_b6": (1.8, 2.6, 0.5, 528), "efficientnet_b7": (2.0, 3.1, 0.5, 600)}
INPUT_SIZE = {name: v[3] for name, v in _VARIANTS.items()}


class ConvBNAct(nn.Sequential):
    """conv + BN + activation (torchvision's ``Conv2dNormActivation``: keys ``.0`` conv, ``.1`` BN); ``silu`` False is the
    linear projection, whose BN may add a residual scaled per sample (stochastic depth)."""

    def __init__(self, cin, cout, kernel_size, stride=1, groups=1, silu=True, bn_eps=1e-5, bn_momentum=0.1):
        super().__init__(Conv2d(cin, cout, kernel_size, stride, (kernel_size - 1) // 2, groups=groups),
                         BatchNorm2d(cout, eps=bn_eps, momentum=bn_momentum))
        self.silu = silu

    def forward(self, x, residual=None, sample_scale=None):
        return conv_bn(x, self[0], self[1], relu=False, residual=residual, silu=self.silu, sample_scale=sample_scale)


class SqueezeExcitation(nn.Module):
    """torchvision's ``SqueezeExcitation(C, C', activation=SiLU)``: keys ``fc1`` / ``fc2`` (1x1 convs with bias)."""

    def __init__(self, channels, squeeze):
        super().__init__()
        self.fc1 = Conv2d(channels, squeeze, 1, bias=True)
        self.fc2 = Conv2d(squeeze, channels, 1, bias=True)

    def forward(self, x):
        return ops.squeeze_excite(x, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias, gate="sigmoid",
                                  act="silu")


class MBConv(nn.Module):
    def __init__(self, expand_ratio, kernel, stride, inp, oup, sd_prob, bn):
        super().__init__()
        if stride not in (1, 2):
            raise ValueError(f"illegal stride value {stride}")
        self.use_res_connect = stride == 1 and inp == oup
        exp = _make_divisible(inp * expand_ratio, 8)
        layers = [ConvBNAct(inp, exp, 1, **bn)] if exp != inp else []
        layers.append(ConvBNAct(exp, exp, kernel, stride, groups=exp, **bn))
        layers.append(SqueezeExcitation(exp, max(1, inp // 4)))
        layers.append(ConvBNAct(exp, oup, 1, silu=False, **bn))
        self.block = nn.Sequential(*layers)
        self.sd_prob = sd_prob          # torchvision's StochasticDepth(p, "row"): no parameters, no state_dict entry
        self.out_channels = oup

    def forward(self, x):
        h = x
        for m in self.block[:-1]:
            h = m(h)
        if not self.use_res_connect:
            return self.block[-1](h)
        keep = None
        if self.training and self.sd_prob > 0.0:
            keep = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
        # z = BN(project(h)) * keep[n] + x in the projection's BN kernel
        return self.block[-1](h, residual=x, sample_scale=keep)


class EfficientNet(nn.Module):
    def __init__(self, width_mult, depth_mult, dropout, input_size, num_classes=1000, stochastic_depth_prob=0.2,
                 bn_eps=1e-5, bn_momentum=0.1):
        super().__init__()
        self.num_classes = num_classes
        self.input_size = input_size
        bn = {"bn_eps": bn_eps, "bn_momentum": bn_momentum}

        def width(c):
            return _make_divisible(c * width_mult, 8)

        stages = [(e, k, s, width(i), width(o), int(math.ceil(n * depth_mult))) for e, k, s, i, o, n in _STAGES]
        features = [ConvBNAct(3, stages[0][3], 3, 2, **bn)]
        total, idx = sum(st[5] for st in stages), 0
        for e, k, s, i, o, n in stages:
            blocks = []
            for j in range(n):
                blocks.append(MBConv(e, k, s if j == 0 else 1, i if j == 0 else o, o,
                                     stochastic_depth_prob * float(idx) / total, bn))
                idx += 1
            features.append(nn.Sequential(*blocks))
        last_in = stages[-1][4]
        self.last_channel = 4 * last_in
        features.append(ConvBNAct(last_in, self.last_channel, 1, **bn))
        self.features = nn.Sequential(*features)
        self.classifier = nn.Sequential(_Dropout(dropout), Linear(self.last_channel, num_classes))
        for m in self.modules():
            if isinstance(m, Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
            elif isinstance(m, Linear):
                r = 1.0 / math.sqrt(m.out_features)
                nn.init.uniform_(m.weight, -r, r)
                nn.init.zeros_(m.bias)

    def forward(self, x):
        x = prepare_input(x)
        x = self.features(x)
        x = ops.global_avg_pool(x)
        x = self.classifier[0](x)
        return self.classifier[1](x)[:, : self.num_classes]


def _efficientnet(name, num_classes=1000, stochastic_depth_prob=0.2, dropout=None, **kw):
    w, d, p, size = _VARIANTS[name]
    if name in ("efficientnet_b5", "efficientnet_b6", "efficientnet_b7"):      # torchvision's BN for B5-B7
        kw.setdefault("bn_eps", 1e-3)
        kw.setdefault("bn_momentum", 0.01)
    return EfficientNet(w, d, p if dropout is None else dropout, size, num_classes=num_classes,
                        stochastic_depth_prob=stochastic_depth_prob, **kw)


def efficientnet_b0(**kw):
    return _efficientnet("efficientnet_b0", **kw)


def efficientnet_b1(**kw):
    return _efficientnet("efficientnet_b1", **kw)


def efficientnet_b2(**kw):
    return _efficientnet("efficientnet_b2", **kw)


def efficientnet_b3(**kw):
    return _efficientnet("efficientnet_b3", **kw)


def efficientnet_b4(**kw):
    return _efficientnet("efficientnet_b4", **kw)


def efficientnet_b5(**kw):
    return _efficientnet("efficientnet_b5", **kw)


def efficientnet_b6(**kw):
    return _efficientnet("efficientnet_b6", **kw)


def efficientnet_b7(**kw):
    return _efficientnet("efficientnet_b7", **kw)
