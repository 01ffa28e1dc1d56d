"""MaxViT-T (keys, key order, shapes and initialisation match ``torchvision.models.maxvit_t``).

Activations are NHWC ([N, C, H, W] channels_last).  The stem is a 3x3 stride-2 conv + BN + GELU (the fused BN with
GELU), then a 3x3 conv with bias.  Each of the 11 ``MaxVitLayer`` is an MBConv, a window-partition attention layer and a
grid-partition attention layer:

* MBConv: BN (no activation), 1x1 expand + BN + GELU, depthwise 3x3 (stride 2 in a block's first layer) + BN + GELU,
  sigmoid / SiLU squeeze-excitation, 1x1 conv + bias; the shortcut is the identity, or 3x3/s2 average pooling + a 1x1
  conv + bias.  Stochastic depth + residual is one kernel in each direction (``ops.maxvit.stochastic_depth_add``).
* Each attention layer is one autograd node (``ops.maxvit_attention_layer``), the Swin block's node with the partition
  attention kernels (csrc/ops/window_attention.cu).  Two independent stochastic-depth draws per layer, one per residual.

The classifier is global average pooling, LayerNorm, Linear, tanh and a bias-free Linear: torchvision's order.
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..ops.maxvit import PARTITION
from ..ops.swin import relative_position_index
from .layers import BatchNorm2d, Conv2d, LayerNorm, Linear, conv_bn, prepare_input

_BN = {"eps": 1e-3, "momentum": 0.01}
_EPS = 1e-5
_HEAD_DIM = 32


def _conv_out(n: int) -> int:
    return (n - 3 + 2) // 2 + 1          # 3x3, stride 2, padding 1


class _ConvNorm(nn.Sequential):
    """torchvision's ``Conv2dNormActivation`` with BN: keys ``.0`` conv, ``.1`` BN; the activation is GELU."""

    def __init__(self, cin, cout, stride=1, groups=1, kernel=3):
        super().__init__(Conv2d(cin, cout, kernel, stride, (kernel - 1) // 2, groups=groups), BatchNorm2d(cout, **_BN))

    def forward(self, x):
        return conv_bn(x, self[0], self[1], relu=False, gelu=True)


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
    """torchvision's MaxViT ``MBConv`` (expansion 4, squeeze ratio 0.25 of the output width): keys ``proj`` (``.1`` the
    1x1 conv after the average pool, or ``.0`` without one) and ``layers.pre_norm`` / ``conv_a`` / ``conv_b`` /
    ``squeeze_excitation`` / ``conv_c``."""

    def __init__(self, cin, cout, stride, sd_prob):
        super().__init__()
        self.stride = stride
        if stride != 1 or cin != cout:
            conv = Conv2d(cin, cout, 1, bias=True)
            self.proj = nn.Sequential(nn.Identity(), conv) if stride == 2 else nn.Sequential(conv)
        else:
            self.proj = None
        mid = 4 * cout
        self.layers = nn.ModuleDict(OrderedDict(
            pre_norm=BatchNorm2d(cin, **_BN), conv_a=_ConvNorm(cin, mid, kernel=1),
            conv_b=_ConvNorm(mid, mid, stride, groups=mid), squeeze_excitation=SqueezeExcitation(mid, cout // 4),
            conv_c=Conv2d(mid, cout, 1, bias=True)))
        self.sd_prob = sd_prob          # torchvision's StochasticDepth(p, "row"): no parameters, no state_dict entry

    def forward(self, x):
        res = x
        if self.proj is not None:
            if self.stride == 2:
                res = ops.avg_pool2d(res, 3, 2, 1)
            res = self.proj[-1](res)
        ly = self.layers
        bn = ly["pre_norm"]
        h = ops.batch_norm_act(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum, relu=False,
                               training=bn.training)
        h = ly["conv_c"](ly["squeeze_excitation"](ly["conv_b"](ly["conv_a"](h))))
        keep = None
        if self.training and self.sd_prob > 0.0:
            keep = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
        return ops.maxvit.stochastic_depth_add(h, res, keep)


class RelativePositionalMultiHeadAttention(nn.Module):
    """Parameter holder with torchvision's state_dict: ``to_qkv`` [3C, C] + bias, ``merge`` [C, C] + bias,
    ``relative_position_bias_table`` [169, heads] (trunc_normal, std 0.02) and the int64 buffer
    ``relative_position_index`` [49, 49]."""

    def __init__(self, dim, heads):
        super().__init__()
        self.n_heads = heads
        self.to_qkv = Linear(dim, 3 * dim)
        self.merge = Linear(dim, dim)
        self.relative_position_bias_table = nn.Parameter(torch.empty((2 * PARTITION - 1) ** 2, heads))
        self.register_buffer("relative_position_index", relative_position_index(PARTITION).view(PARTITION ** 2, -1))
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)


class PartitionAttentionLayer(nn.Module):
    """torchvision's ``PartitionAttentionLayer``: ``attn_layer`` (``.0`` LayerNorm, ``.1`` attention, ``.2`` dropout)
    and ``mlp_layer`` (``.0`` LayerNorm, ``.1`` / ``.3`` the MLP linears, ratio 4)."""

    def __init__(self, dim, partition, sd_prob):
        super().__init__()
        self.partition = partition
        self.attn_layer = nn.Sequential(LayerNorm(dim, eps=_EPS),
                                        RelativePositionalMultiHeadAttention(dim, dim // _HEAD_DIM), nn.Identity())
        self.mlp_layer = nn.Sequential(LayerNorm(dim, eps=_EPS), Linear(dim, 4 * dim), nn.Identity(),
                                       Linear(4 * dim, dim), nn.Identity())
        self.sd_prob = sd_prob

    def forward(self, x):
        n1, a = self.attn_layer[0], self.attn_layer[1]
        n2, m1, m2 = self.mlp_layer[0], self.mlp_layer[1], self.mlp_layer[3]
        keep1 = keep2 = None
        if self.training and self.sd_prob > 0.0:
            keep1 = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
            keep2 = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
        return ops.maxvit_attention_layer(x, self.partition, a.n_heads, n1.eps, n1.weight, n1.bias, a.to_qkv.weight,
                                          a.to_qkv.bias, a.merge.weight, a.merge.bias, a.relative_position_bias_table,
                                          n2.weight, n2.bias, m1.weight, m1.bias, m2.weight, m2.bias, keep1, keep2)


class MaxVitLayer(nn.Module):
    def __init__(self, cin, cout, stride, sd_prob):
        super().__init__()
        self.layers = nn.ModuleDict(OrderedDict(
            MBconv=MBConv(cin, cout, stride, sd_prob), window_attention=PartitionAttentionLayer(cout, "window", sd_prob),
            grid_attention=PartitionAttentionLayer(cout, "grid", sd_prob)))

    def forward(self, x):
        for m in self.layers.values():
            x = m(x)
        return x


class MaxVitBlock(nn.Module):
    def __init__(self, cin, cout, sd_probs):
        super().__init__()
        self.layers = nn.ModuleList(MaxVitLayer(cin if i == 0 else cout, cout, 2 if i == 0 else 1, p)
                                    for i, p in enumerate(sd_probs))

    def forward(self, x):
        for m in self.layers:
            x = m(x)
        return x


class _Stem(nn.Sequential):
    """``.0`` 3x3 stride-2 conv + BN + GELU, ``.1.0`` 3x3 conv with bias."""

    def __init__(self, dim):
        super().__init__(_ConvNorm(3, dim, 2), nn.Sequential(Conv2d(dim, dim, 3, 1, 1, bias=True)))

    def forward(self, x):
        return self[1][0](self[0](x))


class MaxVit(nn.Module):
    def __init__(self, stem_channels, block_channels, block_layers, num_classes=1000, stochastic_depth_prob=0.2,
                 input_size=224):
        super().__init__()
        size = _conv_out(input_size)
        for i in range(len(block_channels)):
            size = _conv_out(size)
            if size % PARTITION != 0:
                raise ValueError(f"input_size {input_size}: the map of block {i} is {size} x {size}, not a multiple of "
                                 f"the partition size {PARTITION}")
        self.num_classes = num_classes
        self.input_size = input_size
        self.stem = _Stem(stem_channels)
        p = np.linspace(0, stochastic_depth_prob, sum(block_layers)).tolist()
        self.blocks = nn.ModuleList()
        cin, idx = stem_channels, 0
        for cout, n in zip(block_channels, block_layers):
            self.blocks.append(MaxVitBlock(cin, cout, p[idx:idx + n]))
            cin, idx = cout, idx + n
        c = block_channels[-1]
        self.classifier = nn.Sequential(nn.Identity(), nn.Identity(), LayerNorm(c, eps=_EPS), Linear(c, c),
                                        nn.Identity(), Linear(c, num_classes, bias=False))
        for m in self.modules():
            if isinstance(m, (Conv2d, Linear)):
                nn.init.normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def forward(self, x):
        x = prepare_input(x)
        x = self.stem(x)
        for b in self.blocks:
            x = b(x)
        x = self.classifier[2](ops.global_avg_pool(x))
        x = ops.maxvit.tanh(self.classifier[3](x))
        return self.classifier[5](x)[:, : self.num_classes]


def maxvit_t(num_classes=1000, stochastic_depth_prob=0.2, input_size=224, mlp_dropout=0.0, attention_dropout=0.0):
    if mlp_dropout != 0.0 or attention_dropout != 0.0:
        raise ValueError("mlp_dropout / attention_dropout inside the MaxViT layers are not supported (only 0.0)")
    return MaxVit(64, [64, 128, 256, 512], [2, 2, 5, 2], num_classes=num_classes,
                  stochastic_depth_prob=stochastic_depth_prob, input_size=input_size)
