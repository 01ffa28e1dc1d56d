"""Swin Transformer V2 Swin-V2-T, -S and -B (keys, key order, shapes and initialisation match
``torchvision.models.swin_v2_t``, ``swin_v2_s`` and ``swin_v2_b``).

Activations are NHWC ([N, C, H, W] channels_last, i.e. torchvision's [N, H, W, C] rows).  The stem and the classifier
are Swin V1's.  Every ``SwinTransformerBlockV2`` (window 8, scaled-cosine attention with a per-head ``logit_scale``, the
continuous position-bias MLP ``cpb_mlp``, post-norm residuals) is one autograd node (``ops.swin_v2_block``); every
``PatchMergingV2`` is another (``ops.patch_merging_v2``: 2x2 gather, the bias-free reduction GEMM, then LayerNorm over
2C).  Window 8 does not divide the 28, 14 and 7 stage maps of a 224 input: the attention kernels handle those padded
maps natively.  ``input_size`` is 256, torchvision's crop for these weights.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from ..ops.swin import relative_position_index
from ..ops.swin_v2 import relative_coords_table
from .layers import LayerNorm, Linear, prepare_input
from .swin import _Stem

# variant -> (embed dim, depths, heads, default stochastic-depth probability) as in torchvision 0.26
_VARIANTS = {"swin_v2_t": (96, (2, 2, 6, 2), (3, 6, 12, 24), 0.2),
             "swin_v2_s": (96, (2, 2, 18, 2), (3, 6, 12, 24), 0.3),
             "swin_v2_b": (128, (2, 2, 18, 2), (4, 8, 16, 32), 0.5)}
_EPS = 1e-5
_WINDOW = 8
INPUT_SIZE = 256


class ShiftedWindowAttentionV2(nn.Module):
    """Parameter holder with torchvision's ``ShiftedWindowAttentionV2`` state_dict: ``logit_scale`` [heads, 1, 1]
    (ln 10), the persistent buffers ``relative_coords_table`` [1, 2w-1, 2w-1, 2] fp32 and ``relative_position_index``
    int64 [w^4], ``qkv`` [3C, C] + bias, ``proj`` [C, C] + bias and ``cpb_mlp`` (``.0`` [512, 2] + bias, ``.1`` ReLU,
    ``.2`` [heads, 512] without bias)."""

    def __init__(self, dim, num_heads, window_size, shift_size):
        super().__init__()
        self.window_size, self.shift_size, self.num_heads = window_size, shift_size, num_heads
        self.logit_scale = nn.Parameter(torch.log(10 * torch.ones((num_heads, 1, 1))))
        self.register_buffer("relative_coords_table", relative_coords_table(window_size))
        self.register_buffer("relative_position_index", relative_position_index(window_size))
        self.qkv = Linear(dim, 3 * dim)
        self.proj = Linear(dim, dim)
        self.cpb_mlp = nn.Sequential(Linear(2, 512), nn.ReLU(inplace=True), Linear(512, num_heads, bias=False))


class SwinTransformerBlockV2(nn.Module):
    """torchvision's ``SwinTransformerBlockV2``: ``norm1``, ``attn``, ``norm2``, ``mlp.0`` / ``mlp.3``; the norms follow
    the attention and the MLP (post-norm).  Stochastic depth draws two independent keep vectors, one per residual
    branch."""

    def __init__(self, dim, num_heads, window_size, shift_size, sd_prob):
        super().__init__()
        self.norm1 = LayerNorm(dim, eps=_EPS)
        self.attn = ShiftedWindowAttentionV2(dim, num_heads, window_size, shift_size)
        self.norm2 = LayerNorm(dim, eps=_EPS)
        self.mlp = nn.Sequential(Linear(dim, 4 * dim), nn.Identity(), nn.Identity(), Linear(4 * dim, dim), nn.Identity())
        self.sd_prob = sd_prob

    def forward(self, x):
        a, m = self.attn, self.mlp
        keep1 = keep2 = None
        if self.training and self.sd_prob > 0.0:
            keep1 = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
            keep2 = ops.stochastic_depth_keep(x.shape[0], self.sd_prob, x.device)
        return ops.swin_v2_block(x, a.num_heads, a.window_size, a.shift_size, self.norm1.eps, a.relative_coords_table,
                                 a.logit_scale, a.qkv.weight, a.qkv.bias, a.proj.weight, a.proj.bias,
                                 a.cpb_mlp[0].weight, a.cpb_mlp[0].bias, a.cpb_mlp[2].weight, self.norm1.weight,
                                 self.norm1.bias, m[0].weight, m[0].bias, m[3].weight, m[3].bias, self.norm2.weight,
                                 self.norm2.bias, keep1, keep2)


class PatchMergingV2(nn.Module):
    """torchvision's ``PatchMergingV2``: ``reduction`` [2C, 4C] without bias, then ``norm`` over 2C (applied after)."""

    def __init__(self, dim):
        super().__init__()
        self.reduction = Linear(4 * dim, 2 * dim, bias=False)
        self.norm = LayerNorm(2 * dim, eps=_EPS)

    def forward(self, x):
        return ops.patch_merging_v2(x, self.reduction.weight, self.norm.weight, self.norm.bias, self.norm.eps)


class SwinTransformerV2(nn.Module):
    def __init__(self, embed_dim, depths, num_heads, num_classes=1000, stochastic_depth_prob=0.1):
        super().__init__()
        self.num_classes = num_classes
        self.input_size = INPUT_SIZE
        layers = [_Stem(embed_dim)]
        total, idx = sum(depths), 0
        for i, (d, h) in enumerate(zip(depths, num_heads)):
            dim = embed_dim * 2 ** i
            blocks = []
            for j in range(d):
                blocks.append(SwinTransformerBlockV2(dim, h, _WINDOW, 0 if j % 2 == 0 else _WINDOW // 2,
                                                     stochastic_depth_prob * float(idx) / (total - 1)))
                idx += 1
            layers.append(nn.Sequential(*blocks))
            if i + 1 < len(depths):
                layers.append(PatchMergingV2(dim))
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


def _swin_v2(name, num_classes=1000, stochastic_depth_prob=None, dropout=0.0, attention_dropout=0.0):
    if dropout != 0.0 or attention_dropout != 0.0:
        raise ValueError("dropout / attention_dropout inside the Swin V2 blocks are not supported (only 0.0)")
    dim, depths, heads, p = _VARIANTS[name]
    return SwinTransformerV2(dim, depths, heads, num_classes=num_classes,
                             stochastic_depth_prob=p if stochastic_depth_prob is None else stochastic_depth_prob)


def swin_v2_t(**kw):
    return _swin_v2("swin_v2_t", **kw)


def swin_v2_s(**kw):
    return _swin_v2("swin_v2_s", **kw)


def swin_v2_b(**kw):
    return _swin_v2("swin_v2_b", **kw)

