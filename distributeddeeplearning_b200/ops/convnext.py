"""ConvNeXt's ops: LayerNorm over the channels of NHWC activations, and the whole CNBlock as ONE autograd node.

    forward   y1 = dw7(x) + b_dw;  t = LN(y1);  h = fc1(t) + b1;  g = gelu(h);  y2 = fc2(g) + b2
              z  = ls[c] * y2 * keep[n] + x
    backward  dy2 = dz * ls * keep   (+ dls, db2 in the same pass)          dg = dgrad_fc2(dy2)   wgrad_fc2 (side stream)
              dh  = dg * gelu'(h)    (+ db1)                                dt = dgrad_fc1(dh)    wgrad_fc1 (side stream)
              dy1 = LN_bwd(dt)       (+ dgamma, dbeta)
              dx  = dgrad_dw7(dy1) + dz                                     <- the '+' is the dgrad's store
              wgrad_dw7 (+ db_dw)

The residual gradient dz rides in the depthwise data gradient, so the block's input gradient is written once and
autograd never sums two gradients of x.  fc1 / fc2 are torchvision's ``nn.Linear`` on the channels-last rows, i.e. 1x1
conv-GEMMs on the existing kernels (their [out, in] weights are the GEMM operand as they are).  The composite of torch
ops is the CPU path and the float64 oracle of the tests; the maths is exactly torchvision's ``CNBlock``.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from . import native
from .functional import CL, grad_buffer, notify_ready, run_wgrad, use_native, weight_bf16


def _dense(x: torch.Tensor) -> bool:
    return x.is_contiguous(memory_format=CL) if x.dim() == 4 else x.is_contiguous()


# ------------------------------------------------------------------------------------------------
# LayerNorm over channels (stem, downsample layers, classifier)
# ------------------------------------------------------------------------------------------------
class _LayerNormChannels(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, train):
        y, mean, rstd = native.layer_norm_fwd(x, weight, bias, eps)
        ctx.params = (weight, bias)
        if train:
            ctx.save_for_backward(x, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        weight, bias = ctx.params
        x, mean, rstd = ctx.saved_tensors
        if not _dense(dy):
            dy = dy.contiguous(memory_format=CL) if dy.dim() == 4 else dy.contiguous()
        dx = native.layer_norm_bwd(dy, x, mean, rstd, weight, grad_buffer(weight) if weight.requires_grad else None,
                                   grad_buffer(bias) if bias.requires_grad else None)
        for p in (weight, bias):
            if p.requires_grad:
                notify_ready(p)
        return (dx if ctx.needs_input_grad[0] else None), None, None, None, None


def layer_norm_channels(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """LayerNorm over the channels of an activation [N, C, H, W] (torchvision's ``LayerNorm2d``) or of a matrix [N, C]
    (``nn.LayerNorm(C)``).  Native for bf16 NHWC activations / contiguous matrices whose width
    ``native.supports_layer_norm`` accepts; the composite is the CPU path."""
    c = x.shape[1]
    if use_native(x) and x.dtype == torch.bfloat16 and x.dim() in (2, 4) and native.supports_layer_norm(c) \
            and _dense(x):
        train = torch.is_grad_enabled() and any(t.requires_grad for t in (x, weight, bias))
        return _LayerNormChannels.apply(x, weight, bias, eps, train)
    w, b = (weight.to(x.dtype), bias.to(x.dtype)) if x.is_cuda else (weight, bias)
    if x.dim() == 2:
        return F.layer_norm(x, (c,), w, b, eps)
    y = F.layer_norm(x.permute(0, 2, 3, 1), (c,), w, b, eps).permute(0, 3, 1, 2)
    return y.contiguous(memory_format=CL) if x.is_cuda else y


# ------------------------------------------------------------------------------------------------
# the ConvNeXt block
# ------------------------------------------------------------------------------------------------
class _ConvNeXtBlock(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, keep, train, eps, dw_w, dw_b, ln_w, ln_b, w1, b1, w2, b2, ls):
        C = x.shape[1]
        wd = weight_bf16(dw_w, groups=C)                               # [C, 49]
        w1b, w2b = weight_bf16(w1), weight_bf16(w2)                     # [4C, C], [C, 4C]
        y1 = native.dwconv7_fwd(x, wd, dw_b)
        t, mean, rstd = native.layer_norm_fwd(y1, ln_w, ln_b, eps)
        h = native.conv_fwd(t, w1b, (1, 1), 1, 0, bias=b1, cout=w1.shape[0])
        g = native.gelu_fwd(h)
        y2 = native.conv_fwd(g, w2b, (1, 1), 1, 0, bias=b2, cout=C)
        z = native.layer_scale_fwd(y2, ls, keep, x)
        ctx.params = (dw_w, dw_b, ln_w, ln_b, w1, b1, w2, b2, ls)
        ctx.keep = keep
        if train:
            ctx.wb = (wd, w1b, w2b)       # views of the bf16 weight arena: see functional._ConvBnAct
            ctx.save_for_backward(x, y1, t, mean, rstd, h, g, y2)
        return z

    @staticmethod
    def backward(ctx, dz):
        dw_w, dw_b, ln_w, ln_b, w1, b1, w2, b2, ls = ctx.params
        x, y1, t, mean, rstd, h, g, y2 = ctx.saved_tensors
        wd, w1b, w2b = ctx.wb
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)

        def gb(p):
            return grad_buffer(p) if p.requires_grad else None

        dy2 = native.layer_scale_bwd(dz, y2, ls, ctx.keep, gb(ls), gb(b2))
        dg = native.conv_dgrad(dy2, w2b, g.shape, (1, 1), 1, 0)
        if w2.requires_grad:
            gw2 = grad_buffer(w2)
            run_wgrad(w2, lambda: native.conv_wgrad(g, dy2, gw2, (1, 1), 1, 0), g, dy2)
        dh = native.gelu_bwd(dg, h, gb(b1))
        dt = native.conv_dgrad(dh, w1b, t.shape, (1, 1), 1, 0)
        if w1.requires_grad:
            gw1 = grad_buffer(w1)
            run_wgrad(w1, lambda: native.conv_wgrad(t, dh, gw1, (1, 1), 1, 0), t, dh)
        dy1 = native.layer_norm_bwd(dt, y1, mean, rstd, ln_w, gb(ln_w), gb(ln_b))
        dx = native.dwconv7_dgrad(dy1, wd, add=dz) if ctx.needs_input_grad[0] else None
        if dw_w.requires_grad or dw_b.requires_grad:
            # a frozen depthwise weight with a trainable bias: the kernel's weight sums go to a scratch slot
            gw = grad_buffer(dw_w) if dw_w.requires_grad else torch.zeros_like(dw_w, memory_format=CL)
            gbias = gb(dw_b)
            run_wgrad(dw_w, lambda: native.dwconv7_wgrad(x, dy1, gw, gbias), x, dy1)
        for p in (ls, b2, w2, b1, w1, ln_w, ln_b, dw_b, dw_w):      # LAST, as in functional._ConvBnAct
            if p.requires_grad:
                notify_ready(p)
        return (dx,) + (None,) * 12


def convnext_block_native(x: torch.Tensor, dw_w: torch.Tensor, w1: torch.Tensor) -> bool:
    """Whether :func:`convnext_block` runs on the native node for this input and these weights."""
    c = x.shape[1]
    return (use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)
            and native.supports_depthwise7(c, tuple(dw_w.shape[2:]), 1, 3, 1, c) and dw_w.shape[1] == 1
            and dw_w.is_contiguous(memory_format=CL) and native.supports_layer_norm(c)
            and native.supports_conv(c, w1.shape[0]) and native.supports_conv(w1.shape[0], c))


def convnext_block(x: torch.Tensor, dw_w: torch.Tensor, dw_b: torch.Tensor, ln_w: torch.Tensor, ln_b: torch.Tensor,
                   eps: float, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor, ls: torch.Tensor,
                   keep: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torchvision's ``CNBlock``: x + keep[n] * ls * fc2(gelu(fc1(LN(dw7(x))))) with the depthwise 7x7 ``dw_w``
    [C, 1, 7, 7] + ``dw_b``, the LayerNorm ``ln_w`` / ``ln_b`` / ``eps``, the linears ``w1`` [4C, C] + ``b1`` and
    ``w2`` [C, 4C] + ``b2``, and the layer scale ``ls`` ([C, 1, 1] or [C]).  ``keep``: fp32 [N] stochastic-depth scales
    (``stochastic_depth_keep``), None in eval or when the drop probability is 0."""
    C = x.shape[1]
    if convnext_block_native(x, dw_w, w1):
        params = (dw_w, dw_b, ln_w, ln_b, w1, b1, w2, b2, ls)
        train = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        return _ConvNeXtBlock.apply(x, keep, train, eps, *params)
    dt = x.dtype if x.is_cuda else dw_w.dtype

    def c(p):
        return p.to(dt) if x.is_cuda else p

    y = F.conv2d(x, c(dw_w), c(dw_b), 1, 3, 1, C)
    y = F.layer_norm(y.permute(0, 2, 3, 1), (C,), c(ln_w), c(ln_b), eps)
    y = F.linear(F.gelu(F.linear(y, c(w1), c(b1))), c(w2), c(b2)).permute(0, 3, 1, 2)
    y = c(ls).reshape(C, 1, 1) * y
    if keep is not None:
        y = y * keep.to(y.dtype).view(-1, 1, 1, 1)
    z = y + x
    return z.contiguous(memory_format=CL) if x.is_cuda else z
