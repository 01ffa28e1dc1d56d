"""ShuffleNetV2 x0.5, x1.0, x1.5 and x2.0 (keys, shapes and initialisation match
``torchvision.models.shufflenet_v2_x0_5`` ... ``shufflenet_v2_x2_0``).

The stem is conv 3x3/s2 + BN + ReLU + max-pool 3x3/s2 (``conv_bn_pool``), then three stages of units
(torchvision's ``InvertedResidual``) and ``conv5`` (1x1 + BN + ReLU, a ``conv_bn`` unit), the mean over the image and
``fc``.  Every unit runs as one autograd node (``ops.shuffle_unit``): its branch BN, concat and channel shuffle are one
kernel pass, and on CUDA units hand each other the two channel halves of their output, so no channel slice is copied;
the last unit of a stage writes its output whole.  x1.0 (58 / 116) and x2.0 (122 / 244) have branch widths that are not
multiples of 8; the node pads them with zero channels internally (see ``ops/shufflenet.py``).  torchvision 0.26 gives
the model no custom initialisation: convolutions keep PyTorch's kaiming-uniform default, BN ones / zeros, the
classifier ``Linear``'s default.
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, conv_bn_pool, prepare_input

# stage output widths (conv1, stage2, stage3, stage4, conv5) of torchvision 0.26; stage repeats 4 / 8 / 4
_WIDTHS = {
    "shufflenet_v2_x0_5": [24, 48, 96, 192, 1024],
    "shufflenet_v2_x1_0": [24, 116, 232, 464, 1024],
    "shufflenet_v2_x1_5": [24, 176, 352, 704, 1024],
    "shufflenet_v2_x2_0": [24, 244, 488, 976, 2048],
}
_REPEATS = [4, 8, 4]


class InvertedResidual(nn.Module):
    """torchvision's unit: ``branch1`` (stride 2 only) = depthwise 3x3 + BN, 1x1 + BN + ReLU; ``branch2`` = 1x1 + BN +
    ReLU, depthwise 3x3 + BN, 1x1 + BN + ReLU.  ``whole_output``: the unit ends its stage and returns its output as one
    tensor (on the native node, a unit inside a stage returns the (lo, hi) halves)."""

    def __init__(self, inp, oup, stride, whole_output=False):
        super().__init__()
        if not 1 <= stride <= 3:
            raise ValueError("illegal stride value")
        self.stride = stride
        bf = oup // 2
        if stride == 1 and inp != bf << 1:
            raise ValueError("Invalid combination of stride and inp / oup")
        if stride > 1:
            self.branch1 = nn.Sequential(Conv2d(inp, inp, 3, stride, 1, groups=inp), BatchNorm2d(inp),
                                         Conv2d(inp, bf, 1), BatchNorm2d(bf), nn.ReLU(inplace=True))
        else:
            self.branch1 = nn.Sequential()
        self.branch2 = nn.Sequential(Conv2d(inp if stride > 1 else bf, bf, 1), BatchNorm2d(bf), nn.ReLU(inplace=True),
                                     Conv2d(bf, bf, 3, stride, 1, groups=bf), BatchNorm2d(bf),
                                     Conv2d(bf, bf, 1), BatchNorm2d(bf), nn.ReLU(inplace=True))
        self.whole_output = whole_output

    def forward(self, x):
        b1 = [self.branch1[i] for i in range(4)] if self.stride > 1 else None
        b2 = [self.branch2[i] for i in (0, 1, 3, 4, 5, 6)]
        return ops.shuffle_unit(x, b1, b2, self.whole_output)


class ShuffleNetV2(nn.Module):
    def __init__(self, name, num_classes=1000):
        super().__init__()
        widths = _WIDTHS[name]
        self.num_classes = num_classes
        self.input_size = 224
        self.conv1 = nn.Sequential(Conv2d(3, widths[0], 3, 2, 1), BatchNorm2d(widths[0]), nn.ReLU(inplace=True))
        inp = widths[0]
        for i, (reps, oup) in enumerate(zip(_REPEATS, widths[1:4])):
            units = [InvertedResidual(inp, oup, 2)]
            units += [InvertedResidual(oup, oup, 1) for _ in range(reps - 1)]
            units[-1].whole_output = True
            setattr(self, f"stage{i + 2}", nn.Sequential(*units))
            inp = oup
        self.conv5 = nn.Sequential(Conv2d(inp, widths[-1], 1), BatchNorm2d(widths[-1]), nn.ReLU(inplace=True))
        self.fc = Linear(widths[-1], num_classes)

    def forward(self, x):
        x = prepare_input(x)
        x = conv_bn_pool(x, self.conv1[0], self.conv1[1], 3, 2, 1)
        x = self.stage2(x)
        x = self.stage3(x)
        x = self.stage4(x)
        x = conv_bn(x, self.conv5[0], self.conv5[1])
        x = ops.global_avg_pool(x)
        return self.fc(x)[:, : self.num_classes]


def _shufflenet_v2(name, **kw):
    """torchvision 0.26's builder argument: ``num_classes``."""
    unknown = sorted(set(kw) - {"num_classes"})
    if unknown:
        raise ValueError(f"{name}: unexpected arguments {unknown}")
    return ShuffleNetV2(name, **kw)


def shufflenet_v2_x0_5(**kw):
    return _shufflenet_v2("shufflenet_v2_x0_5", **kw)


def shufflenet_v2_x1_0(**kw):
    return _shufflenet_v2("shufflenet_v2_x1_0", **kw)


def shufflenet_v2_x1_5(**kw):
    return _shufflenet_v2("shufflenet_v2_x1_5", **kw)


def shufflenet_v2_x2_0(**kw):
    return _shufflenet_v2("shufflenet_v2_x2_0", **kw)
