"""MNASNet-B1 0.5 / 0.75 / 1.0 / 1.3 (keys, shapes and initialisation match ``torchvision.models.mnasnet*``).

Every layer is a fused ``conv_bn`` unit: the stem conv, the 3x3 / 5x5 depthwise convolutions at stride 1 and 2 (the
stencil kernels of csrc/ops/depthwise*.cu) and the 1x1 GEMMs, with ReLU (not ReLU6).  A block's projection BN has no
activation and adds the block input inside the BN kernel when the block keeps its shape, as in MobileNetV2.
torchvision's ``_get_depths`` rounds every width to a multiple of 8, which keeps every layer on the native kernels.
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input
from .mobilenet import _Dropout

# the paper's TensorFlow momentum 0.9997 in PyTorch's convention
_BN_MOMENTUM = 1 - 0.9997


class _InvertedResidual(nn.Module):
    def __init__(self, in_ch, out_ch, kernel_size, stride, expansion_factor, bn_momentum=0.1):
        super().__init__()
        if stride not in (1, 2):
            raise ValueError(f"stride should be 1 or 2 instead of {stride}")
        if kernel_size not in (3, 5):
            raise ValueError(f"kernel_size should be 3 or 5 instead of {kernel_size}")
        mid = in_ch * expansion_factor
        self.apply_residual = in_ch == out_ch and stride == 1
        # the ReLU entries hold no parameters: they keep torchvision's indices (and so its state_dict keys)
        self.layers = nn.Sequential(
            Conv2d(in_ch, mid, 1), BatchNorm2d(mid, momentum=bn_momentum), nn.ReLU(inplace=True),
            Conv2d(mid, mid, kernel_size, stride, kernel_size // 2, groups=mid), BatchNorm2d(mid, momentum=bn_momentum),
            nn.ReLU(inplace=True),
            Conv2d(mid, out_ch, 1), BatchNorm2d(out_ch, momentum=bn_momentum))

    def forward(self, x):
        m = self.layers
        h = conv_bn(conv_bn(x, m[0], m[1], relu=True), m[3], m[4], relu=True)
        return conv_bn(h, m[6], m[7], relu=False, residual=x if self.apply_residual else None)


def _stack(in_ch, out_ch, kernel_size, stride, exp_factor, repeats, bn_momentum):
    first = _InvertedResidual(in_ch, out_ch, kernel_size, stride, exp_factor, bn_momentum)
    rest = [_InvertedResidual(out_ch, out_ch, kernel_size, 1, exp_factor, bn_momentum) for _ in range(1, repeats)]
    return nn.Sequential(first, *rest)


def _round_to_multiple_of(val: float, divisor: int, round_up_bias: float = 0.9) -> int:
    """torchvision's asymmetric rounding: up, unless ``val`` is at most 10 % above the lower multiple."""
    new_val = max(divisor, int(val + divisor / 2) // divisor * divisor)
    return new_val if new_val >= round_up_bias * val else new_val + divisor


def _get_depths(alpha: float):
    return [_round_to_multiple_of(d * alpha, 8) for d in (32, 16, 24, 40, 80, 96, 192, 320)]


class MNASNet(nn.Module):
    input_size = 224
    # torchvision reads this from the checkpoint's metadata: version 1 means the fixed-width stem of the first release,
    # which would not load at alpha != 1.0
    _version = 2

    def __init__(self, alpha: float, num_classes=1000, dropout=0.2):
        super().__init__()
        if alpha <= 0.0:
            raise ValueError(f"alpha should be greater than 0.0 instead of {alpha}")
        self.alpha, self.num_classes = alpha, num_classes
        d = _get_depths(alpha)
        m = _BN_MOMENTUM
        self.layers = nn.Sequential(
            Conv2d(3, d[0], 3, 2, 1), BatchNorm2d(d[0], momentum=m), nn.ReLU(inplace=True),
            Conv2d(d[0], d[0], 3, 1, 1, groups=d[0]), BatchNorm2d(d[0], momentum=m), nn.ReLU(inplace=True),
            Conv2d(d[0], d[1], 1), BatchNorm2d(d[1], momentum=m),
            _stack(d[1], d[2], 3, 2, 3, 3, m), _stack(d[2], d[3], 5, 2, 3, 3, m), _stack(d[3], d[4], 5, 2, 6, 3, m),
            _stack(d[4], d[5], 3, 1, 6, 2, m), _stack(d[5], d[6], 5, 2, 6, 4, m), _stack(d[6], d[7], 3, 1, 6, 1, m),
            Conv2d(d[7], 1280, 1), BatchNorm2d(1280, momentum=m), nn.ReLU(inplace=True))
        self.classifier = nn.Sequential(_Dropout(dropout), Linear(1280, num_classes))
        for mod in self.modules():
            if isinstance(mod, Conv2d):
                nn.init.kaiming_normal_(mod.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(mod, BatchNorm2d):
                nn.init.ones_(mod.weight)
                nn.init.zeros_(mod.bias)
            elif isinstance(mod, Linear):
                nn.init.kaiming_uniform_(mod.weight, mode="fan_out", nonlinearity="sigmoid")
                nn.init.zeros_(mod.bias)

    def forward(self, x):
        m = self.layers
        x = prepare_input(x)
        x = conv_bn(x, m[0], m[1], relu=True)
        x = conv_bn(x, m[3], m[4], relu=True)
        x = conv_bn(x, m[6], m[7], relu=False)
        for i in range(8, 14):
            x = m[i](x)
        x = conv_bn(x, m[14], m[15], relu=True)
        x = ops.global_avg_pool(x)
        x = self.classifier[0](x)
        return self.classifier[1](x)[:, : self.num_classes]


def mnasnet0_5(num_classes=1000, **kw):
    return MNASNet(0.5, num_classes=num_classes, **kw)


def mnasnet0_75(num_classes=1000, **kw):
    return MNASNet(0.75, num_classes=num_classes, **kw)


def mnasnet1_0(num_classes=1000, **kw):
    return MNASNet(1.0, num_classes=num_classes, **kw)


def mnasnet1_3(num_classes=1000, **kw):
    return MNASNet(1.3, num_classes=num_classes, **kw)
