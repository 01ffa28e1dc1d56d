"""Swin Transformer Swin-T, -S and -B (V1; keys, key order, shapes and initialisation match ``torchvision.models.swin_t``,
``swin_s`` and ``swin_b``).

Activations are NHWC ([N, C, H, W] channels_last, i.e. torchvision's [N, H, W, C] rows).  The stem (a 4x4 stride-4 conv
with bias, then LayerNorm over channels) is ConvNeXt's.  Every ``SwinTransformerBlock`` is one autograd node
(``ops.swin_block``) around the shifted-window attention kernels; every ``PatchMerging`` is another
(``ops.patch_merging``: 2x2 gather + LayerNorm over 4C, then the bias-free reduction GEMM).  The classifier applies
``norm`` to the NHWC rows, then the global average pool, then ``head``: torchvision's order.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..ops.swin import relative_position_index
from .layers import Conv2d, LayerNorm, Linear, prepare_input

# variant -> (embed dim, depths, heads, default stochastic-depth probability) as in torchvision 0.26
_VARIANTS = {"swin_t": (96, (2, 2, 6, 2), (3, 6, 12, 24), 0.2),
             "swin_s": (96, (2, 2, 18, 2), (3, 6, 12, 24), 0.3),
             "swin_b": (128, (2, 2, 18, 2), (4, 8, 16, 32), 0.5)}
_EPS = 1e-5
_WINDOW = 7


class ShiftedWindowAttention(nn.Module):
    """Parameter holder with torchvision's ``ShiftedWindowAttention`` state_dict: ``relative_position_bias_table``
    [(2w-1)^2, heads] (trunc_normal, std 0.02), the persistent int64 buffer ``relative_position_index`` [w^4],
    ``qkv`` [3C, C] + bias and ``proj`` [C, C] + bias."""

    def __init__(self, dim, num_heads, window_size, shift_size):
        super().__init__()
        self.window_size, self.shift_size, self.num_heads = window_size, shift_size, num_heads
        self.qkv = Linear(dim, 3 * dim)
        self.proj = Linear(dim, dim)
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * window_size - 1) ** 2, num_heads))
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)
        self.register_buffer("relative_position_index", relative_position_index(window_size))


class SwinTransformerBlock(nn.Module):
    """torchvision's ``SwinTransformerBlock``: ``norm1``, ``attn``, ``norm2``, ``mlp.0`` / ``mlp.3`` (``.1`` GELU and
    ``.2`` / ``.4`` dropout hold no parameters).  Stochastic depth draws two independent keep vectors, one per residual
    branch."""

    def __init__(self, dim, num_heads, window_size, shift_size, sd_prob):
        super().__init__()
        self.norm1 = LayerNorm(dim, eps=_EPS)
        self.attn = ShiftedWindowAttention(dim, num_heads, window_size, shift_size)
        self.norm2 = LayerNorm(dim, eps=_EPS)
        self.mlp = nn.Sequential(Linear(dim, 4 * dim), nn.Identity(), nn.Identity(), Linear(4 * dim, dim), nn.Identity())
        self.sd_prob = sd_prob          # torchvision's StochasticDepth(p, "row"): no parameters, no state_dict entry

    def forward(self, x):
        a, m = self.attn, self.mlp
        keep1 = keep2 = None
        if self.training and self.sd_prob > 0.0:
            keep1 = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
            keep2 = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
        return ops.swin_block(x, a.num_heads, a.window_size, a.shift_size, self.norm1.eps, self.norm1.weight,
                              self.norm1.bias, a.qkv.weight, a.qkv.bias, a.proj.weight, a.proj.bias,
                              a.relative_position_bias_table, self.norm2.weight, self.norm2.bias, m[0].weight, m[0].bias,
                              m[3].weight, m[3].bias, keep1, keep2)


class PatchMerging(nn.Module):
    """torchvision's ``PatchMerging``: ``reduction`` [2C, 4C] without bias, then ``norm`` over 4C (applied first)."""

    def __init__(self, dim):
        super().__init__()
        self.reduction = Linear(4 * dim, 2 * dim, bias=False)
        self.norm = LayerNorm(4 * dim, eps=_EPS)

    def forward(self, x):
        return ops.patch_merging(x, self.norm.weight, self.norm.bias, self.norm.eps, self.reduction.weight)


class _Stem(nn.Sequential):
    """``.0`` the 4x4 stride-4 conv with bias, ``.2`` LayerNorm over channels (``.1`` is torchvision's Permute)."""

    def __init__(self, dim):
        super().__init__(Conv2d(3, dim, 4, 4, bias=True), nn.Identity(), LayerNorm(dim, eps=_EPS))

    def forward(self, x):
        return self[2](self[0](x))


class SwinTransformer(nn.Module):
    def __init__(self, embed_dim, depths, num_heads, num_classes=1000, stochastic_depth_prob=0.1):
        super().__init__()
        self.num_classes = num_classes
        self.input_size = 224
        layers = [_Stem(embed_dim)]
        total, idx = sum(depths), 0
        for i, (d, h) in enumerate(zip(depths, num_heads)):
            dim = embed_dim * 2 ** i
            blocks = []
            for j in range(d):
                blocks.append(SwinTransformerBlock(dim, h, _WINDOW, 0 if j % 2 == 0 else _WINDOW // 2,
                                                   stochastic_depth_prob * float(idx) / (total - 1)))
                idx += 1
            layers.append(nn.Sequential(*blocks))
            if i + 1 < len(depths):
                layers.append(PatchMerging(dim))
        self.features = nn.Sequential(*layers)
        num_features = embed_dim * 2 ** (len(depths) - 1)
        self.norm = LayerNorm(num_features, eps=_EPS)
        self.head = Linear(num_features, num_classes)
        for m in self.modules():
            if isinstance(m, Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def forward(self, x):
        x = prepare_input(x)
        x = self.features(x)
        x = self.norm(x)
        x = ops.global_avg_pool(x)
        return self.head(x)[:, : self.num_classes]


def _swin(name, num_classes=1000, stochastic_depth_prob=None, dropout=0.0, attention_dropout=0.0):
    if dropout != 0.0 or attention_dropout != 0.0:
        raise ValueError("dropout / attention_dropout inside the Swin blocks are not supported (only 0.0)")
    dim, depths, heads, p = _VARIANTS[name]
    return SwinTransformer(dim, depths, heads, num_classes=num_classes,
                           stochastic_depth_prob=p if stochastic_depth_prob is None else stochastic_depth_prob)


def swin_t(**kw):
    return _swin("swin_t", **kw)


def swin_s(**kw):
    return _swin("swin_s", **kw)


def swin_b(**kw):
    return _swin("swin_b", **kw)
