"""Vision Transformer ViT-B/16, -B/32, -L/16 and -L/32 (keys, key order, shapes and initialisation match
``torchvision.models.vit_b_16`` ... ``vit_l_32``).

The patch embedding (a P x P stride-P conv with bias, the class token and the position embedding) is one autograd node
(``ops.vit_embed``): patchify, the conv as a GEMM on the conv-GEMM kernels, token assembly.  Every encoder block is one
autograd node (``ops.vit_encoder_block``) around the fused attention kernels.  The classifier takes the class-token rows
first and applies ``encoder.ln`` to them ([N, C]; LayerNorm is per row, so this is torchvision's maths), then
``heads.head``.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .. import ops
from .layers import Conv2d, LayerNorm, Linear, prepare_input

# variant -> (patch, layers, heads, hidden, mlp) as in torchvision 0.26
_VARIANTS = {"vit_b_16": (16, 12, 12, 768, 3072), "vit_b_32": (32, 12, 12, 768, 3072),
             "vit_l_16": (16, 24, 16, 1024, 4096), "vit_l_32": (32, 24, 16, 1024, 4096)}


class MultiheadAttention(nn.Module):
    """Parameter holder with ``nn.MultiheadAttention``'s state_dict (packed ``in_proj_weight`` [3C, C] /
    ``in_proj_bias``, ``out_proj``) and its initialisation."""

    def __init__(self, dim, num_heads):
        super().__init__()
        self.embed_dim, self.num_heads = dim, num_heads
        self.in_proj_weight = nn.Parameter(torch.empty(3 * dim, dim))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * dim))
        self.out_proj = Linear(dim, dim)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.zeros_(self.out_proj.bias)


class MLPBlock(nn.Sequential):
    """torchvision's ``MLPBlock``: ``.0`` / ``.3`` the linears (``.1`` GELU, ``.2`` / ``.4`` dropout hold no parameters),
    xavier-uniform weights and normal(std 1e-6) biases."""

    def __init__(self, dim, mlp_dim):
        super().__init__(Linear(dim, mlp_dim), nn.Identity(), nn.Identity(), Linear(mlp_dim, dim), nn.Identity())
        for m in (self[0], self[3]):
            nn.init.xavier_uniform_(m.weight)
            nn.init.normal_(m.bias, std=1e-6)


class EncoderBlock(nn.Module):
    def __init__(self, num_heads, dim, mlp_dim):
        super().__init__()
        self.num_heads = num_heads
        self.ln_1 = LayerNorm(dim, eps=1e-6)
        self.self_attention = MultiheadAttention(dim, num_heads)
        self.ln_2 = LayerNorm(dim, eps=1e-6)
        self.mlp = MLPBlock(dim, mlp_dim)

    def forward(self, x):
        a, m = self.self_attention, self.mlp
        return ops.vit_encoder_block(x, self.num_heads, self.ln_1.eps, self.ln_1.weight, self.ln_1.bias,
                                     a.in_proj_weight, a.in_proj_bias, a.out_proj.weight, a.out_proj.bias,
                                     self.ln_2.weight, self.ln_2.bias, m[0].weight, m[0].bias, m[3].weight, m[3].bias)


class Encoder(nn.Module):
    def __init__(self, seq_length, num_layers, num_heads, dim, mlp_dim):
        super().__init__()
        self.pos_embedding = nn.Parameter(torch.empty(1, seq_length, dim).normal_(std=0.02))
        self.layers = nn.Sequential()
        for i in range(num_layers):
            self.layers.add_module(f"encoder_layer_{i}", EncoderBlock(num_heads, dim, mlp_dim))
        self.ln = LayerNorm(dim, eps=1e-6)


class _Heads(nn.Module):
    def __init__(self, dim, num_classes):
        super().__init__()
        self.head = Linear(dim, num_classes)
        nn.init.zeros_(self.head.weight)
        nn.init.zeros_(self.head.bias)


class VisionTransformer(nn.Module):
    def __init__(self, image_size, patch_size, num_layers, num_heads, hidden_dim, mlp_dim, num_classes=1000):
        super().__init__()
        if image_size % patch_size != 0:
            raise ValueError(f"image_size {image_size} is not a multiple of the patch size {patch_size}")
        self.image_size, self.patch_size, self.hidden_dim = image_size, patch_size, hidden_dim
        self.num_classes = num_classes
        self.input_size = image_size
        self.class_token = nn.Parameter(torch.zeros(1, 1, hidden_dim))
        self.conv_proj = Conv2d(3, hidden_dim, patch_size, stride=patch_size, bias=True)
        nn.init.trunc_normal_(self.conv_proj.weight, std=math.sqrt(1.0 / (3 * patch_size * patch_size)))
        nn.init.zeros_(self.conv_proj.bias)
        seq_length = (image_size // patch_size) ** 2 + 1
        self.seq_length = seq_length
        self.encoder = Encoder(seq_length, num_layers, num_heads, hidden_dim, mlp_dim)
        self.heads = _Heads(hidden_dim, num_classes)

    def forward(self, x):
        if x.shape[-2] != self.image_size or x.shape[-1] != self.image_size:
            raise ValueError(f"expected {self.image_size}x{self.image_size} images, got {tuple(x.shape[-2:])}")
        x = prepare_input(x)
        x = ops.vit_embed(x, self.conv_proj.weight, self.conv_proj.bias, self.class_token,
                          self.encoder.pos_embedding, self.patch_size)
        x = self.encoder.layers(x)
        x = x[:, 0].contiguous()
        x = self.encoder.ln(x)
        return self.heads.head(x)[:, : self.num_classes]


def _vit(name, image_size=224, num_classes=1000, dropout=0.0, attention_dropout=0.0, representation_size=None,
         conv_stem_configs=None):
    if dropout != 0.0 or attention_dropout != 0.0:
        raise ValueError("dropout / attention_dropout inside the encoder are not supported (only 0.0)")
    if representation_size is not None:
        raise ValueError("representation_size (a pre-logits layer) is not supported")
    if conv_stem_configs is not None:
        raise ValueError("conv_stem_configs (a convolutional stem) is not supported")
    patch, layers, heads, hidden, mlp = _VARIANTS[name]
    return VisionTransformer(image_size, patch, layers, heads, hidden, mlp, num_classes=num_classes)


def vit_b_16(**kw):
    return _vit("vit_b_16", **kw)


def vit_b_32(**kw):
    return _vit("vit_b_32", **kw)


def vit_l_16(**kw):
    return _vit("vit_l_16", **kw)


def vit_l_32(**kw):
    return _vit("vit_l_32", **kw)
