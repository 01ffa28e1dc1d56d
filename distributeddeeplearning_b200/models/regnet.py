"""RegNetX and RegNetY (400MF to 32GF, and RegNetY-128GF), as ``torchvision.models.regnet_*``.

The block widths come from the quantised linear rule of the RegNet paper (``BlockParams.from_init_params`` in
torchvision: depth, w_0, w_a, w_m, group width), computed here in the same float32 arithmetic, so every model has
torchvision's ``state_dict`` key for key.  A block is ``ResBottleneckBlock``: 1x1 conv + BN + ReLU, grouped 3x3 with the
stride + BN + ReLU, (RegNetY) a squeeze-excitation with a ReLU inner activation and a sigmoid gate, 1x1 conv + BN, plus
the identity or a 1x1 projection, then ReLU.  On the native training path each block is one ``ops.residual_block`` node
(the grouped 3x3 on the group-bundle mode of the conv kernels, ``ops.native.grouped_conv_native``); in eval and on the
CPU the fused units and the torch composite of the SE run instead.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .. import ops
from ..ops.blocks import residual_block, residual_block_supported
from ..ops.functional import squeeze_excite_composite
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input

# name -> (depth, w_0, w_a, w_m, group width, SE ratio) as in torchvision 0.26
_PARAMS = {
    "regnet_y_400mf": (16, 48, 27.89, 2.09, 8, 0.25),
    "regnet_y_800mf": (14, 56, 38.84, 2.4, 16, 0.25),
    "regnet_y_1_6gf": (27, 48, 20.71, 2.65, 24, 0.25),
    "regnet_y_3_2gf": (21, 80, 42.63, 2.66, 24, 0.25),
    "regnet_y_8gf": (17, 192, 76.82, 2.19, 56, 0.25),
    "regnet_y_16gf": (18, 200, 106.23, 2.48, 112, 0.25),
    "regnet_y_32gf": (20, 232, 115.89, 2.53, 232, 0.25),
    "regnet_y_128gf": (27, 456, 160.83, 2.52, 264, 0.25),
    "regnet_x_400mf": (22, 24, 24.48, 2.54, 16, None),
    "regnet_x_800mf": (16, 56, 35.73, 2.28, 16, None),
    "regnet_x_1_6gf": (18, 80, 34.01, 2.25, 24, None),
    "regnet_x_3_2gf": (25, 88, 26.31, 2.25, 48, None),
    "regnet_x_8gf": (23, 80, 49.56, 2.88, 120, None),
    "regnet_x_16gf": (22, 216, 55.59, 2.1, 128, None),
    "regnet_x_32gf": (23, 320, 69.86, 2.0, 168, None),
}


def _make_divisible(v, divisor):
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return new_v + divisor if new_v < 0.9 * v else new_v


def block_params(depth, w_0, w_a, w_m, group_width):
    """[(depth, width, group width)] of the four stages (every stage starts with a stride-2 block), from the
    quantised linear width rule: block j has width w_0 * w_m ** round(log(u_j / w_0) / log(w_m)) rounded to a multiple
    of 8, u_j = w_0 + w_a * j; consecutive equal widths form a stage; a stage's group width is at most its width, and
    its width is rounded to a multiple of the group width."""
    widths_cont = torch.arange(depth) * w_a + w_0
    capacity = torch.round(torch.log(widths_cont / w_0) / math.log(w_m))
    widths = (torch.round(torch.divide(w_0 * torch.pow(w_m, capacity), 8)) * 8).int().tolist()
    stages = []
    for w in widths:
        if stages and stages[-1][1] == w:
            stages[-1][0] += 1
        else:
            stages.append([1, w])
    out = []
    for d, w in stages:
        g = min(group_width, w)
        out.append((d, _make_divisible(w, g), g))
    return out


def grouped_shapes(name=None, size=224):
    """Distinct grouped 3x3 layers (groups > 1) of one RegNet (``name``) or of all 15 at ``size`` as (C, H_in, stride,
    group width): every stage starts with a stride-2 block on a map of size / 2 ** (stage + 1)."""
    out = set()
    for n, prm in _PARAMS.items():
        if name is not None and n != name:
            continue
        h = size // 2
        for d, w, g in block_params(*prm[:5]):
            if w > g:                  # one group (w == g) is a dense convolution
                out.add((w, h, 2, g))
                if d > 1:
                    out.add((w, (h + 1) // 2, 1, g))
            h = (h + 1) // 2
    return sorted(out)


def _conv_norm(cin, cout, kernel, stride=1, groups=1):
    return nn.Sequential(Conv2d(cin, cout, kernel, stride, (kernel - 1) // 2, groups=groups), BatchNorm2d(cout))


class SqueezeExcitation(nn.Module):
    """torchvision's ``SqueezeExcitation(C, C', activation=ReLU)``: keys ``fc1`` / ``fc2`` (1x1 convs with bias),
    sigmoid gate."""

    def __init__(self, channels, squeeze):
        super().__init__()
        self.fc1 = Conv2d(channels, squeeze, 1, bias=True)
        self.fc2 = Conv2d(squeeze, channels, 1, bias=True)

    def forward(self, x):
        return squeeze_excite_composite(x, self.fc1.weight, self.fc1.bias, self.fc2.weight, self.fc2.bias, "sigmoid",
                                        "relu")


class BottleneckTransform(nn.Module):
    def __init__(self, width_in, width_out, stride, group_width, se_ratio):
        super().__init__()
        self.a = _conv_norm(width_in, width_out, 1)
        self.b = _conv_norm(width_out, width_out, 3, stride, width_out // group_width)
        if se_ratio:
            self.se = SqueezeExcitation(width_out, int(round(se_ratio * width_in)))
        self.c = _conv_norm(width_out, width_out, 1)


class ResBottleneckBlock(nn.Module):
    def __init__(self, width_in, width_out, stride, group_width, se_ratio):
        super().__init__()
        self.proj = _conv_norm(width_in, width_out, 1, stride) if width_in != width_out or stride != 1 else None
        self.f = BottleneckTransform(width_in, width_out, stride, group_width, se_ratio)

    def forward(self, x):
        f = self.f
        convs, bns = (f.a[0], f.b[0], f.c[0]), (f.a[1], f.b[1], f.c[1])
        se = getattr(f, "se", None)
        ds = (self.proj[0], self.proj[1]) if self.proj is not None else None
        if residual_block_supported(x, convs, bns, ds, se):
            return residual_block(x, convs, bns, ds, se=se)       # one autograd node, SE inside
        h = conv_bn(x, f.a[0], f.a[1], relu=True)
        h = conv_bn(h, f.b[0], f.b[1], relu=True)
        if se is not None:
            h = se(h)
        identity = conv_bn(x, self.proj[0], self.proj[1], relu=False) if self.proj is not None else x
        return conv_bn(h, f.c[0], f.c[1], relu=True, residual=identity)


class RegNet(nn.Module):
    input_size = 224

    def __init__(self, depth, w_0, w_a, w_m, group_width, se_ratio=None, num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.stem = _conv_norm(3, 32, 3, 2)
        stages = []
        width_in = 32
        for i, (d, w, g) in enumerate(block_params(depth, w_0, w_a, w_m, group_width)):
            blocks = nn.Sequential()
            for j in range(d):
                blocks.add_module(f"block{i + 1}-{j}",
                                  ResBottleneckBlock(width_in if j == 0 else w, w, 2 if j == 0 else 1, g, se_ratio))
            stages.append((f"block{i + 1}", blocks))
            width_in = w
        self.trunk_output = nn.Sequential()
        for name, s in stages:
            self.trunk_output.add_module(name, s)
        self.fc = Linear(width_in, num_classes)
        for m in self.modules():
            if isinstance(m, Conv2d):
                fan_out = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                nn.init.normal_(m.weight, mean=0.0, std=math.sqrt(2.0 / fan_out))
        nn.init.normal_(self.fc.weight, mean=0.0, std=0.01)
        nn.init.zeros_(self.fc.bias)

    def forward(self, x):
        x = prepare_input(x)
        x = conv_bn(x, self.stem[0], self.stem[1], relu=True)
        x = self.trunk_output(x)
        x = ops.global_avg_pool(x)
        return self.fc(x)[:, : self.num_classes]


def _builder(name):
    def build(**kw):
        num_classes = kw.pop("num_classes", 1000)
        if kw:
            raise ValueError(f"{name}: unsupported arguments {sorted(kw)} (only num_classes)")
        return RegNet(*_PARAMS[name], num_classes=num_classes)

    build.__name__ = build.__qualname__ = name
    build.__doc__ = f"torchvision's ``{name}``."
    return build


regnet_y_400mf = _builder("regnet_y_400mf")
regnet_y_800mf = _builder("regnet_y_800mf")
regnet_y_1_6gf = _builder("regnet_y_1_6gf")
regnet_y_3_2gf = _builder("regnet_y_3_2gf")
regnet_y_8gf = _builder("regnet_y_8gf")
regnet_y_16gf = _builder("regnet_y_16gf")
regnet_y_32gf = _builder("regnet_y_32gf")
regnet_y_128gf = _builder("regnet_y_128gf")
regnet_x_400mf = _builder("regnet_x_400mf")
regnet_x_800mf = _builder("regnet_x_800mf")
regnet_x_1_6gf = _builder("regnet_x_1_6gf")
regnet_x_3_2gf = _builder("regnet_x_3_2gf")
regnet_x_8gf = _builder("regnet_x_8gf")
regnet_x_16gf = _builder("regnet_x_16gf")
regnet_x_32gf = _builder("regnet_x_32gf")
