"""ConvNeXt-Tiny / -Small / -Base / -Large (keys, shapes and initialisation match ``torchvision.models.convnext_tiny`` ...
``convnext_large``).

The stem (4x4 stride-4 conv with bias) and the downsample convs (2x2 stride 2 with bias) run on the conv-GEMM kernels
through ``conv_bias_act``; their LayerNorms, and the classifier's on the pooled [N, C] rows, on the native LayerNorm over
channels.  Every CNBlock is one autograd node (``ops.convnext_block``): depthwise 7x7 + bias, LayerNorm, fc1 + GELU,
fc2, then layer scale, stochastic depth and the residual add in one kernel.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from .layers import Conv2d, LayerNorm, Linear, prepare_input

# variant -> (stage widths, stage depths, default stochastic-depth probability) as in torchvision 0.26
_VARIANTS = {"convnext_tiny": ((96, 192, 384, 768), (3, 3, 9, 3), 0.1),
             "convnext_small": ((96, 192, 384, 768), (3, 3, 27, 3), 0.4),
             "convnext_base": ((128, 256, 512, 1024), (3, 3, 27, 3), 0.5),
             "convnext_large": ((192, 384, 768, 1536), (3, 3, 27, 3), 0.5)}


class CNBlock(nn.Module):
    """torchvision's ``CNBlock``: ``block.0`` depthwise 7x7 conv with bias, ``block.2`` LayerNorm, ``block.3`` / ``block.5``
    the linears (``block.1`` / ``.4`` / ``.6`` are the parameter-free Permute / GELU / Permute), ``layer_scale`` [C, 1, 1]."""

    def __init__(self, dim, layer_scale, sd_prob):
        super().__init__()
        self.block = nn.Sequential(Conv2d(dim, dim, 7, padding=3, groups=dim, bias=True), nn.Identity(),
                                   LayerNorm(dim, eps=1e-6), Linear(dim, 4 * dim), nn.Identity(), Linear(4 * dim, dim),
                                   nn.Identity())
        self.layer_scale = nn.Parameter(torch.ones(dim, 1, 1) * layer_scale)
        self.sd_prob = sd_prob          # torchvision's StochasticDepth(p, "row"): no parameters, no state_dict entry

    def forward(self, x):
        dw, ln, fc1, fc2 = self.block[0], self.block[2], self.block[3], self.block[5]
        keep = None
        if self.training and self.sd_prob > 0.0:
            keep = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
        return ops.convnext_block(x, dw.weight, dw.bias, ln.weight, ln.bias, ln.eps, fc1.weight, fc1.bias, fc2.weight,
                                  fc2.bias, self.layer_scale, keep)


class _ConvLN(nn.Sequential):
    """The stem: ``.0`` conv with bias, ``.1`` LayerNorm over channels (torchvision's ``Conv2dNormActivation``)."""

    def __init__(self, cin, cout, k, stride):
        super().__init__(Conv2d(cin, cout, k, stride, bias=True), LayerNorm(cout, eps=1e-6))

    def forward(self, x):
        return self[1](self[0](x))


class _LNConv(nn.Sequential):
    """A downsample layer: ``.0`` LayerNorm over channels, ``.1`` 2x2 stride-2 conv with bias."""

    def __init__(self, cin, cout):
        super().__init__(LayerNorm(cin, eps=1e-6), Conv2d(cin, cout, 2, 2, bias=True))

    def forward(self, x):
        return self[1](self[0](x))


class ConvNeXt(nn.Module):
    def __init__(self, widths, depths, num_classes=1000, stochastic_depth_prob=0.0, layer_scale=1e-6):
        super().__init__()
        self.num_classes = num_classes
        self.input_size = 224
        layers = [_ConvLN(3, widths[0], 4, 4)]
        total, idx = sum(depths), 0
        for i, (w, d) in enumerate(zip(widths, depths)):
            blocks = []
            for _ in range(d):
                blocks.append(CNBlock(w, layer_scale, stochastic_depth_prob * idx / (total - 1.0)))
                idx += 1
            layers.append(nn.Sequential(*blocks))
            if i + 1 < len(widths):
                layers.append(_LNConv(w, widths[i + 1]))
        self.features = nn.Sequential(*layers)
        self.classifier = nn.Sequential(LayerNorm(widths[-1], eps=1e-6), nn.Identity(), Linear(widths[-1], num_classes))
        for m in self.modules():
            if isinstance(m, (Conv2d, Linear)):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def forward(self, x):
        x = prepare_input(x)
        x = self.features(x)
        x = ops.global_avg_pool(x)
        x = self.classifier[0](x)
        return self.classifier[2](x)[:, : self.num_classes]


def _convnext(name, num_classes=1000, stochastic_depth_prob=None, layer_scale=1e-6):
    widths, depths, p = _VARIANTS[name]
    return ConvNeXt(widths, depths, num_classes=num_classes,
                    stochastic_depth_prob=p if stochastic_depth_prob is None else stochastic_depth_prob,
                    layer_scale=layer_scale)


def convnext_tiny(**kw):
    return _convnext("convnext_tiny", **kw)


def convnext_small(**kw):
    return _convnext("convnext_small", **kw)


def convnext_base(**kw):
    return _convnext("convnext_base", **kw)


def convnext_large(**kw):
    return _convnext("convnext_large", **kw)
