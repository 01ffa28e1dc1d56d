"""EfficientNetV2's residual Fused-MBConv block as ONE autograd node.

    expand 1  forward   y = conv_kxk(x) [+BN stats];  z = silu(BN(y)) * keep[n] + x                    (BN code 6)
              backward  dy = bn_bwd(dz; code 6)                    dx = dgrad_kxk(dy) + dz    wgrad_kxk
    expand e  forward   y1 = conv_kxk(x);  h = silu(BN1(y1));  y2 = conv_1x1(h);  z = BN2(y2) * keep[n] + x
              backward  dy2 = bn_bwd(dz; stochastic depth)         dh = dgrad_1x1(dy2)        wgrad_1x1
                        dy1 = bn_bwd(dh; SiLU)                     dx = dgrad_kxk(dy1) + dz   wgrad_kxk

The '+ dz' is the data gradient's store (``conv_dgrad(..., add=dz)``): the residual's gradient is dz itself, so the
BN backward writes no copy of it and autograd never sums two gradients of x.  ``keep`` is the per-sample
stochastic-depth scale (``stochastic_depth_keep``), None in eval or at drop probability 0.  The maths is exactly
torchvision's ``FusedMBConv`` with ``use_res_connect``; :func:`fused_mbconv_composite` (torch ops) is the CPU path and the
float64 oracle of the tests, and :func:`fused_mbconv_layers` (one ``conv_bn`` unit per layer, the scale and the add as
separate ops) is the path of the shapes the node does not take.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from . import native
from .functional import CL, conv_bn_act, grad_buffer, notify_ready, run_wgrad, use_native, weight_bf16


def _pad(w: torch.Tensor) -> int:
    return (w.shape[2] - 1) // 2


class _FusedMBConv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, keep, training, save, bn_cfg, w1, g1, b1, rm1, rv1, w2, g2, b2, rm2, rv2):
        """bn_cfg: (eps, momentum) of BN1 and, with an expansion, of BN2; w2 / g2 / ... are None without one."""
        k, pad = (w1.shape[2], w1.shape[3]), _pad(w1)
        wb1 = weight_bf16(w1)
        if training:
            y1, st1 = native.conv_fwd(x, wb1, k, 1, pad, stats=True, cout=w1.shape[0])
        else:
            y1, st1 = native.conv_fwd(x, wb1, k, 1, pad, cout=w1.shape[0]), None
        eps1, mom1 = bn_cfg[0]
        if w2 is None:
            z, save1 = native.bn_act_fwd(y1, st1, g1, b1, rm1, rv1, eps1, mom1, 6, x, training, sample_scale=keep)
            saved, wbs = (x, y1, save1), (wb1,)
        else:
            h, save1 = native.bn_act_fwd(y1, st1, g1, b1, rm1, rv1, eps1, mom1, 4, None, training)
            wb2 = weight_bf16(w2)
            if training:
                y2, st2 = native.conv_fwd(h, wb2, (1, 1), 1, 0, stats=True, cout=w2.shape[0])
            else:
                y2, st2 = native.conv_fwd(h, wb2, (1, 1), 1, 0, cout=w2.shape[0]), None
            eps2, mom2 = bn_cfg[1]
            z, save2 = native.bn_act_fwd(y2, st2, g2, b2, rm2, rv2, eps2, mom2, False, x, training, sample_scale=keep)
            saved, wbs = (x, y1, save1, h, y2, save2), (wb1, wb2)
        ctx.params = (w1, g1, b1, w2, g2, b2)
        ctx.keep = keep
        if save:
            ctx.wbs = wbs             # views of the bf16 weight arena: see functional._ConvBnAct
            ctx.save_for_backward(*saved)
        return z

    @staticmethod
    def backward(ctx, dz):
        w1, g1, b1, w2, g2, b2 = ctx.params
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)

        def gb(p):
            return grad_buffer(p) if p.requires_grad else None

        k, pad = (w1.shape[2], w1.shape[3]), _pad(w1)
        if w2 is None:
            x, y1, save1 = ctx.saved_tensors
            dy1, _, _ = native.bn_act_bwd(dz, None, y1, save1, g1, 6, False, gb(g1), gb(b1), beta=b1,
                                          sample_scale=ctx.keep)
            params = (g1, b1, w1)
        else:
            x, y1, save1, h, y2, save2 = ctx.saved_tensors
            dy2, _, _ = native.bn_act_bwd(dz, None, y2, save2, g2, False, False, gb(g2), gb(b2), beta=b2,
                                          sample_scale=ctx.keep)
            dh = native.conv_dgrad(dy2, ctx.wbs[1], h.shape, (1, 1), 1, 0)
            if w2.requires_grad:
                gw2 = grad_buffer(w2)
                run_wgrad(w2, lambda: native.conv_wgrad(h, dy2, gw2, (1, 1), 1, 0), h, dy2)
            dy1, _, _ = native.bn_act_bwd(dh, None, y1, save1, g1, 4, False, gb(g1), gb(b1), beta=b1,
                                          had_residual=False)
            params = (g2, b2, w2, g1, b1, w1)
        dx = native.conv_dgrad(dy1, ctx.wbs[0], x.shape, k, 1, pad, add=dz) if ctx.needs_input_grad[0] else None
        if w1.requires_grad:
            gw1 = grad_buffer(w1)
            run_wgrad(w1, lambda: native.conv_wgrad(x, dy1, gw1, k, 1, pad), x, dy1)
        for p in params:          # LAST, as in functional._ConvBnAct
            if p.requires_grad:
                notify_ready(p)
        return (dx,) + (None,) * 14


def fused_mbconv_supported(x: torch.Tensor, conv1, bn1, conv2=None, bn2=None) -> bool:
    """Whether :func:`fused_mbconv` runs on the native node: a bf16 NHWC input, a stride-1 k x k conv (odd k, 'same'
    padding) keeping the width, or expanding it for a 1x1 projection back, widths the conv and BN kernels take, KRSC
    weights, and BN in training (or no gradient wanted)."""
    c, w1 = x.shape[1], conv1.weight
    if not (use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)):
        return False
    if bn1.training != (bn2.training if bn2 is not None else bn1.training):
        return False
    if not bn1.training and torch.is_grad_enabled():
        return False
    if conv1.groups != 1 or conv1.stride not in (1, (1, 1)) or conv1.dilation not in (1, (1, 1)) \
            or w1.shape[2] != w1.shape[3] or w1.shape[2] % 2 != 1 or w1.shape[1] != c \
            or tuple(native._pad2(conv1.padding)) != (_pad(w1), _pad(w1)) or not w1.is_contiguous(memory_format=CL):
        return False
    e = w1.shape[0]
    if not (native.supports_conv(c, e) and native.bn_supported(e)):
        return False
    if conv2 is None:
        return e == c
    w2 = conv2.weight
    return (conv2.groups == 1 and tuple(w2.shape) == (c, e, 1, 1) and conv2.stride in (1, (1, 1))
            and native.supports_conv(e, c) and native.bn_supported(c))


def fused_mbconv_composite(x, w1, g1, b1, rm1, rv1, eps1, mom1, training, w2=None, g2=None, b2=None, rm2=None, rv2=None,
                           eps2=1e-3, mom2=0.1, keep: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torchvision's residual ``FusedMBConv`` in torch ops: silu(BN1(conv(x))) [-> BN2(conv_1x1(.))], times
    ``keep[n]``, plus x.  On CPU in the weights' dtype, on CUDA in the activations' dtype; a 16-bit activation gets its BN
    in fp32.  In float64 it is the oracle of the tests."""
    dt = x.dtype if x.is_cuda else w1.dtype

    def bn(y, rm, rv, g, b, eps, mom):
        yb = y.float() if y.dtype in (torch.bfloat16, torch.float16) else y
        return F.batch_norm(yb, rm, rv, g, b, training, mom, eps).to(y.dtype)

    y = F.conv2d(x.to(dt), w1.to(dt), None, 1, _pad(w1))
    h = F.silu(bn(y, rm1, rv1, g1, b1, eps1, mom1))
    if w2 is not None:
        h = bn(F.conv2d(h, w2.to(dt)), rm2, rv2, g2, b2, eps2, mom2)
    if keep is not None:
        h = h * keep.to(h.dtype).view(-1, 1, 1, 1)
    return h + x.to(dt)


def fused_mbconv_layers(x: torch.Tensor, conv1, bn1, conv2=None, bn2=None, keep: Optional[torch.Tensor] = None):
    """The block as one ``conv_bn`` unit per layer: without an expansion the scale and the residual add are separate
    elementwise ops (the BN kernels' SiLU takes no residual) and autograd sums the two gradients of x; with one, the
    projection's BN applies both, as in EfficientNet's MBConv."""
    def unit(h, conv, bn, **kw):
        return conv_bn_act(h, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, conv.stride,
                           conv.padding, conv.dilation, bn.eps, bn.momentum, training=bn.training, **kw)

    h = unit(x, conv1, bn1, relu=False, silu=True)
    if conv2 is not None:
        return unit(h, conv2, bn2, relu=False, residual=x, **({"sample_scale": keep} if keep is not None else {}))
    if keep is not None:
        h = h * keep.to(h.dtype).view(-1, 1, 1, 1)
    return h + x


def fused_mbconv(x: torch.Tensor, conv1, bn1, conv2=None, bn2=None, keep: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torchvision's ``FusedMBConv`` with a residual: x + keep[n] * silu(BN1(conv1(x))) without an expansion, or
    x + keep[n] * BN2(conv2(silu(BN1(conv1(x))))) with one (``conv2`` the 1x1 projection).  ``conv1`` / ``conv2`` are
    ``models.layers.Conv2d`` and ``bn1`` / ``bn2`` ``BatchNorm2d`` holders; ``keep``: fp32 [N] stochastic-depth scales
    (``stochastic_depth_keep``), None in eval or when the drop probability is 0.  One native node where
    :func:`fused_mbconv_supported` holds; per-layer ``conv_bn`` units elsewhere on CUDA; the composite on CPU."""
    if fused_mbconv_supported(x, conv1, bn1, conv2, bn2):
        training = bn1.training
        ps = [conv1.weight, bn1.weight, bn1.bias, bn1.running_mean, bn1.running_var]
        ps += [conv2.weight, bn2.weight, bn2.bias, bn2.running_mean, bn2.running_var] if conv2 is not None \
            else [None] * 5
        save = training and torch.is_grad_enabled() and (x.requires_grad or any(
            p is not None and p.requires_grad for p in ps))
        cfg = ((bn1.eps, bn1.momentum),) + (((bn2.eps, bn2.momentum),) if bn2 is not None else ())
        return _FusedMBConv.apply(x, keep if training else None, training, save, cfg, *ps)
    if x.is_cuda:
        return fused_mbconv_layers(x, conv1, bn1, conv2, bn2, keep)
    two = conv2 is not None
    return fused_mbconv_composite(x, conv1.weight, bn1.weight, bn1.bias, bn1.running_mean, bn1.running_var, bn1.eps,
                                  bn1.momentum, bn1.training,
                                  *((conv2.weight, bn2.weight, bn2.bias, bn2.running_mean, bn2.running_var, bn2.eps,
                                     bn2.momentum) if two else ()), keep=keep)
