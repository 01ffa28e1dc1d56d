"""Whole residual block (BasicBlock / Bottleneck) as ONE autograd node.

Why: with one node per conv+BN unit, autograd itself has to sum the two gradients that reach a block's input
(main path + identity/downsample path) with a separate elementwise kernel — 16 extra read-read-write passes over
the largest activations of ResNet-50 per step.  Here the block's backward is written out by hand, and that sum
rides in the epilogue of the first conv's dgrad kernel (``out = acc + add``), so the block input gradient is
produced exactly once.  It also trims Python/autograd overhead (1 node instead of 3-4 per block).

    forward   h0 = x;  y_i = conv_i(h_{i-1}) [+BN stats in the epilogue];  h_i = relu(bn_i(y_i))        i < L
              idn = x  |  bn_d(conv_d(x))
              out = relu(bn_L(y_L) + idn)
    backward  (dy_L, dres) = bn_bwd(dout; mask from out)      d_{L-1} = dgrad_L(dy_L)      wgrad_L
              dy_i = bn_bwd(d_i; mask recomputed from y_i)    d_{i-1} = dgrad_i(dy_i)      wgrad_i
              dx = dgrad_1(dy_1) + (dres | dgrad_d(bn_bwd(dres)))          <- the '+' is the dgrad epilogue

Reference parity: the maths is exactly torchvision's BasicBlock/Bottleneck (SURVEY.md 2.7); this only changes how
the backward is scheduled.
"""
from __future__ import annotations

import os
from typing import Sequence

import torch

from . import native
from .functional import CL, grad_buffer, notify_ready, run_wgrad, weight_bf16


# Folding the BN-backward reduction into the producing dgrad's epilogue removes 32 launches and one read of each inner
# gradient tensor but makes those (already epilogue-bound) dgrads slower.  Off unless DDL_FUSE_BN_REDUCE=1 (not
# re-measured on H100).
FUSE_BN_REDUCE = os.environ.get("DDL_FUSE_BN_REDUCE", "0") != "0"


class _ResidualBlock(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cfg, *params):
        """cfg: tuple of per-layer (stride, pad, dil, eps, momentum) for the L main convs [+ downsample last];
        params: per layer (weight, gamma, beta, running_mean, running_var), downsample (if any) last."""
        n_main, has_ds = cfg["n_main"], cfg["has_ds"]
        layers = [params[5 * i: 5 * i + 5] for i in range(n_main + (1 if has_ds else 0))]
        saved = []
        wbs = []
        h = x
        identity = x
        if has_ds:
            w, g, b, rm, rv = layers[n_main]
            st, pad, dil, eps, mom = cfg["layers"][n_main]
            wb = weight_bf16(w)
            yd, stats = native.conv_fwd(x, wb, (w.shape[2], w.shape[3]), st, pad, dil, stats=True, cout=w.shape[0])
            identity, save_d = native.bn_act_fwd(yd, stats, g, b, rm, rv, eps, mom, False, None, True)
            ds_pack = (yd, save_d, wb)
        for i in range(n_main):
            w, g, b, rm, rv = layers[i]
            st, pad, dil, eps, mom = cfg["layers"][i]
            wb = weight_bf16(w)
            y, stats = native.conv_fwd(h, wb, (w.shape[2], w.shape[3]), st, pad, dil, stats=True, cout=w.shape[0])
            last = i == n_main - 1
            if last:      # residual layer: backward masks with 1 bit per element instead of re-reading the block output
                z, save, zmask = native.bn_act_fwd(y, stats, g, b, rm, rv, eps, mom, True, identity, True, want_mask=True)
            else:
                z, save = native.bn_act_fwd(y, stats, g, b, rm, rv, eps, mom, True, None, True)
            saved += [h, y, save]
            wbs.append(wb)
            h = z
        ctx.cfg = cfg
        ctx.layers = layers
        ctx.wbs = wbs
        ctx.ds_pack = ds_pack if has_ds else None
        ctx.save_for_backward(x, zmask, *saved)
        return h

    @staticmethod
    def backward(ctx, dout):
        cfg, layers = ctx.cfg, ctx.layers
        n_main, has_ds = cfg["n_main"], cfg["has_ds"]
        x, zmask = ctx.saved_tensors[0], ctx.saved_tensors[1]
        saved = ctx.saved_tensors[2:]
        if not dout.is_contiguous(memory_format=CL):
            dout = dout.contiguous(memory_format=CL)
        need_dx = ctx.needs_input_grad[0]
        d = dout
        dres = None
        dx = None
        gated_add = None
        pre = None
        for i in range(n_main - 1, -1, -1):
            w, g, b, _, _ = layers[i]
            st, pad, dil, _, _ = cfg["layers"][i]
            h_in, y, save = saved[3 * i], saved[3 * i + 1], saved[3 * i + 2]
            kernel = (w.shape[2], w.shape[3])
            last = i == n_main - 1
            gg = grad_buffer(g) if g.requires_grad else None
            bg = grad_buffer(b) if b.requires_grad else None
            z = None if last else saved[3 * (i + 1)]           # this layer's output = next layer's input (unused: the
            #                                                    mask is recomputed from y; last layer: bit mask)
            # identity shortcut + a dgrad that can add in its epilogue: the shortcut gradient dout * (out > 0) is
            # formed there from dout and the bit mask, so the BN-backward kernel need not write (and dgrad re-read) it
            gate = last and not has_ds and need_dx and native.dgrad_supports_add(
                (layers[0][0].shape[2], layers[0][0].shape[3]), cfg["layers"][0][0])
            dy, dr, _ = native.bn_act_bwd(d, z, y, save, g, True, last and not gate, gg, bg, beta=b, had_residual=last,
                                          zmask=zmask if last else None, pre_reduced=pre)
            if gate:
                gated_add = (dout, zmask)
            if last:
                dres = dr
            pre = None
            if i > 0:
                # the dgrad that produces d_{i-1} also reduces dbeta / dgamma of BN_{i-1} in its epilogue (it holds the
                # gradient tile anyway and only has to read the y tile): BN_{i-1}'s backward is then one pass, not two
                gp, bp = layers[i - 1][1], layers[i - 1][2]
                pre = native.zeros_f32((2, h_in.shape[1]), h_in.device) if FUSE_BN_REDUCE else None
                d = native.conv_dgrad(dy, ctx.wbs[i], h_in.shape, kernel, st, pad, dil,
                                      bn_reduce=(saved[3 * (i - 1) + 1], gp, bp, saved[3 * (i - 1) + 2], pre)
                                      if pre is not None else None)
            elif need_dx:
                add = dres
                if has_ds:
                    wd, gd, bd, _, _ = layers[n_main]
                    std, padd, dild, _, _ = cfg["layers"][n_main]
                    yd, save_d, wbd = ctx.ds_pack
                    ggd = grad_buffer(gd) if gd.requires_grad else None
                    bgd = grad_buffer(bd) if bd.requires_grad else None
                    dyd, _, _ = native.bn_act_bwd(dres, yd, yd, save_d, gd, False, False, ggd, bgd)
                    add = native.conv_dgrad(dyd, wbd, x.shape, (wd.shape[2], wd.shape[3]), std, padd, dild)
                    if wd.requires_grad:
                        gwd = grad_buffer(wd)
                        run_wgrad(wd, lambda: native.conv_wgrad(x, dyd, gwd, (wd.shape[2], wd.shape[3]), std, padd, dild),
                                  x, dyd)
                    for p in (gd, bd, wd):
                        if p.requires_grad:
                            notify_ready(p)
                if gated_add is not None:
                    dx = native.conv_dgrad(dy, ctx.wbs[0], x.shape, kernel, st, pad, dil, add=gated_add[0],
                                           add_mask=gated_add[1])
                elif native.dgrad_supports_add(kernel, st):
                    dx = native.conv_dgrad(dy, ctx.wbs[0], x.shape, kernel, st, pad, dil, add=add)
                else:
                    dx = native.add(native.conv_dgrad(dy, ctx.wbs[0], x.shape, kernel, st, pad, dil), add)
            if w.requires_grad:
                gw = grad_buffer(w)
                run_wgrad(w, lambda h_in=h_in, dy=dy, gw=gw, kernel=kernel, st=st, pad=pad, dil=dil:
                          native.conv_wgrad(h_in, dy, gw, kernel, st, pad, dil), h_in, dy)
            for p in (g, b, w):
                if p.requires_grad:
                    notify_ready(p)
        if not need_dx and has_ds:
            # block input needs no gradient but the downsample parameters still do
            wd, gd, bd, _, _ = layers[n_main]
            std, padd, dild, _, _ = cfg["layers"][n_main]
            yd, save_d, wbd = ctx.ds_pack
            dyd, _, _ = native.bn_act_bwd(dres, yd, yd, save_d, gd, False, False, grad_buffer(gd), grad_buffer(bd))
            native.conv_wgrad(x, dyd, grad_buffer(wd), (wd.shape[2], wd.shape[3]), std, padd, dild)
            for p in (gd, bd, wd):
                notify_ready(p)
        return (dx, None) + (None,) * (5 * len(layers))


def residual_block_supported(x: torch.Tensor, convs: Sequence, bns: Sequence, downsample) -> bool:
    from .functional import use_native

    if not use_native(x) or not torch.is_grad_enabled():
        return False
    mods = list(zip(convs, bns)) + ([tuple(downsample)] if downsample is not None else [])
    cin = x.shape[1]
    for conv, bn in mods:
        if not bn.training:
            return False
        if not native.supports_conv(conv.in_channels, conv.out_channels) or not native.bn_supported(conv.out_channels):
            return False
        if conv.in_channels <= 4 or not conv.weight.is_contiguous(memory_format=CL) and conv.weight.dim() == 4 and \
                conv.weight.shape[2] * conv.weight.shape[3] > 1:
            return False
    return cin % 8 == 0


def residual_block(x: torch.Tensor, convs: Sequence, bns: Sequence, downsample=None) -> torch.Tensor:
    """convs/bns: the main-path layer containers (``models.layers.Conv2d`` / ``BatchNorm2d``) in order;
    downsample: optional (conv, bn) pair of the projection shortcut."""
    mods = list(zip(convs, bns)) + ([tuple(downsample)] if downsample is not None else [])
    cfg = {"n_main": len(convs), "has_ds": downsample is not None,
           "layers": [(c.stride, c.padding, c.dilation, b.eps, b.momentum) for c, b in mods]}
    params = []
    for c, b in mods:
        params += [c.weight, b.weight, b.bias, b.running_mean, b.running_var]
    return _ResidualBlock.apply(x, cfg, *params)
