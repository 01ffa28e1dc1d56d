"""EfficientNetV2-S, -M and -L (keys, shapes and initialisation match ``torchvision.models.efficientnet_v2_s`` ...
``efficientnet_v2_l``).

The early stages are Fused-MBConv blocks: a k x k conv + BN + SiLU, then, when the block expands, a 1x1 linear projection
+ BN.  A block that keeps its shape adds its input after stochastic depth; it runs as one autograd node
(``ops.fused_mbconv``): without an expansion the BN kernel applies SiLU, the per-sample scale and the residual add
(BN code 6), and in backward the residual's gradient rides in the k x k data gradient's store.  The other Fused blocks are
two ``conv_bn`` units.  The later stages are EfficientNet's MBConv blocks (``models.efficientnet``), and the stem and
head are its ``ConvBNAct`` units.
"""
from __future__ import annotations

import math

import torch.nn as nn

from .. import ops
from .efficientnet import ConvBNAct, MBConv
from .layers import BatchNorm2d, Conv2d, Linear, prepare_input
from .mobilenet import _Dropout, _make_divisible

# (expand ratio, kernel, stride, input channels, output channels, layers) per stage, as in torchvision 0.26: the
# Fused-MBConv stages, then the MBConv stages
_STAGES = {
    "efficientnet_v2_s": ([(1, 3, 1, 24, 24, 2), (4, 3, 2, 24, 48, 4), (4, 3, 2, 48, 64, 4)],
                          [(4, 3, 2, 64, 128, 6), (6, 3, 1, 128, 160, 9), (6, 3, 2, 160, 256, 15)]),
    "efficientnet_v2_m": ([(1, 3, 1, 24, 24, 3), (4, 3, 2, 24, 48, 5), (4, 3, 2, 48, 80, 5)],
                          [(4, 3, 2, 80, 160, 7), (6, 3, 1, 160, 176, 14), (6, 3, 2, 176, 304, 18),
                           (6, 3, 1, 304, 512, 5)]),
    "efficientnet_v2_l": ([(1, 3, 1, 32, 32, 4), (4, 3, 2, 32, 64, 7), (4, 3, 2, 64, 96, 7)],
                          [(4, 3, 2, 96, 192, 10), (6, 3, 1, 192, 224, 19), (6, 3, 2, 224, 384, 25),
                           (6, 3, 1, 384, 640, 7)]),
}
# variant -> (classifier dropout, crop size) as in torchvision 0.26
_VARIANTS = {"efficientnet_v2_s": (0.2, 384), "efficientnet_v2_m": (0.3, 480), "efficientnet_v2_l": (0.4, 480)}
INPUT_SIZE = {name: v[1] for name, v in _VARIANTS.items()}
_LAST_CHANNEL = 1280
_BN = {"bn_eps": 1e-3, "bn_momentum": 0.1}


class FusedMBConv(nn.Module):
    """torchvision's ``FusedMBConv``: ``block.0`` the k x k conv + BN + SiLU, ``block.1`` the 1x1 projection + BN (only
    when the block expands)."""

    def __init__(self, expand_ratio, kernel, stride, inp, oup, sd_prob, bn):
        super().__init__()
        if stride not in (1, 2):
            raise ValueError(f"illegal stride value {stride}")
        self.use_res_connect = stride == 1 and inp == oup
        exp = _make_divisible(inp * expand_ratio, 8)
        if exp != inp:
            layers = [ConvBNAct(inp, exp, kernel, stride, **bn), ConvBNAct(exp, oup, 1, silu=False, **bn)]
        else:
            layers = [ConvBNAct(inp, oup, kernel, stride, **bn)]
        self.block = nn.Sequential(*layers)
        self.sd_prob = sd_prob          # torchvision's StochasticDepth(p, "row"): no parameters, no state_dict entry
        self.out_channels = oup

    def forward(self, x):
        if not self.use_res_connect:
            for m in self.block:
                x = m(x)
            return x
        keep = None
        if self.training and self.sd_prob > 0.0:
            keep = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
        c1 = self.block[0]
        c2 = self.block[1] if len(self.block) > 1 else None
        return ops.fused_mbconv(x, c1[0], c1[1], *((c2[0], c2[1]) if c2 is not None else ()), keep=keep)


class EfficientNetV2(nn.Module):
    def __init__(self, name, dropout, num_classes=1000, stochastic_depth_prob=0.2):
        super().__init__()
        self.num_classes = num_classes
        self.input_size = INPUT_SIZE[name]
        fused, mb = _STAGES[name]
        stages = [(FusedMBConv,) + st for st in fused] + [(MBConv,) + st for st in mb]
        features = [ConvBNAct(3, stages[0][4], 3, 2, **_BN)]
        total, idx = sum(st[6] for st in stages), 0
        for block, e, k, s, i, o, n in stages:
            blocks = []
            for j in range(n):
                blocks.append(block(e, k, s if j == 0 else 1, i if j == 0 else o, o,
                                    stochastic_depth_prob * float(idx) / total, _BN))
                idx += 1
            features.append(nn.Sequential(*blocks))
        self.last_channel = _LAST_CHANNEL
        features.append(ConvBNAct(stages[-1][5], self.last_channel, 1, **_BN))
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


def _efficientnet_v2(name, **kw):
    """torchvision 0.26's builder arguments: ``num_classes``, ``stochastic_depth_prob`` and ``dropout``."""
    unknown = sorted(set(kw) - {"num_classes", "stochastic_depth_prob", "dropout"})
    if unknown:
        raise ValueError(f"{name}: unexpected arguments {unknown}")
    dropout = kw.pop("dropout", _VARIANTS[name][0])
    return EfficientNetV2(name, dropout, **kw)


def efficientnet_v2_s(**kw):
    return _efficientnet_v2("efficientnet_v2_s", **kw)


def efficientnet_v2_m(**kw):
    return _efficientnet_v2("efficientnet_v2_m", **kw)


def efficientnet_v2_l(**kw):
    return _efficientnet_v2("efficientnet_v2_l", **kw)
