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
    where dgrad_1 is a 1x1 conv, its epilogue also takes the previous block's bn_L sums over dx (``_Bn3Handoff``)

An optional squeeze-excitation (RegNetY) sits between the last two layers: h_{L-1} <- h_{L-1} * sigmoid(fc2(relu(
fc1(mean_hw(h_{L-1}))))).  The last dgrad then produces the gradient at the SE output, so it does not take BN_{L-1}'s
reduction (that needs the gradient at the SE input, formed by ``se_apply``).

Reference parity: the maths is exactly torchvision's BasicBlock/Bottleneck (SURVEY.md 2.7); this only changes how
the backward is scheduled.
"""
from __future__ import annotations

from typing import Sequence

import torch

from . import native
from .functional import CL, grad_buffer, notify_ready, run_wgrad, weight_bf16


def _se_fwd(x, w1, b1, w2, b2):
    """x * sigmoid(fc2(relu(fc1(mean_hw(x))))) on the squeeze-excitation kernels; fc1 / fc2 are the 1x1 convs
    [C', C, 1, 1] / [C, C', 1, 1] with biases.  fc1's output h keeps C' rounded up to 64 columns (the pad is zero) and
    is fc2's operand as it stands, against fc2's weight padded with zero columns to match (made here, so a captured
    graph rebuilds it every replay).  Returns y and what :func:`_se_bwd` needs."""
    w1b, w2b = weight_bf16(w1), weight_bf16(w2, stem=False)      # [C', C], [C, C']
    pooled = native.global_avgpool_fwd(x)                         # [N, C]
    h = native.linear_fwd(pooled, w1b, b1, relu=True)             # [N, C' rounded up to 64]
    w2p = w2b if h.shape[1] == w2b.shape[1] else native.pad_cols_bf16(w2b, h.shape[1])
    s = native.linear_fwd(h, w2p, b2)                             # [N, C rounded up to 64]: the gate logits
    return native.se_scale(x, s, gate="sigmoid"), (x, pooled, h, s, w1b, w2p)


def _se_bwd(dy, saved, w1, b1, w2, b2):
    """Input gradient of :func:`_se_fwd` (both paths in one ``se_apply`` pass); accumulates the fc1 / fc2 gradients of
    the parameters that need them."""
    x, pooled, h, s, w1b, w2p = saved
    cs, c = w1.shape[0], w1.shape[1]
    ds = native.se_reduce(dy, x, s, gate="sigmoid")               # [N, C rounded up to 64], pad columns 0
    if b2.requires_grad:
        native.bias_relu_bwd(ds, ds, grad_buffer(b2), False, c_valid=c)
    dh = native.linear_dgrad(ds, w2p)                             # [N, C' rounded up to 64], pad columns 0
    if w2.requires_grad:
        if w2p.shape[1] == cs:
            native.linear_wgrad(h, ds, grad_buffer(w2))
        else:
            gw = native.zeros_f32((c, w2p.shape[1]), ds.device)
            native.linear_wgrad(h, ds, gw)
            native.fold_cols_f32(gw, grad_buffer(w2))
    dh = native.bias_relu_bwd(dh, h, grad_buffer(b1) if b1.requires_grad else None, True, c_valid=cs)
    dx = native.se_apply(dy, s, native.linear_dgrad(dh, w1b), gate="sigmoid")
    if w1.requires_grad:
        native.linear_wgrad(pooled, dh, grad_buffer(w1))
    for p in (b2, w2, b1, w1):
        if p.requires_grad:
            notify_ready(p)
    return dx


class _Bn3Handoff:
    """Lets the next block's first dgrad take the block-output BN's dbeta / dgamma sums.

    The block's forward fills in what that BN's backward reduction reads (its input y, saved mean / invstd, gamma,
    beta and the output's ReLU bit mask).  The next block's backward computes the gradient of that output with a 1x1
    dgrad that also accumulates the sums (``conv_dgrad(..., bn_reduce=...)``) and records the tensor it returned.  This
    block's backward uses the sums only if the gradient it receives is that very tensor, unmodified: had autograd added
    another consumer's gradient, the sums would not describe it, and the stand-alone reduction runs instead."""

    def __init__(self):
        self.bn = None          # (y, save, gamma, beta, zmask) of the block-output BN
        self.sums = None        # fp32 [2, C] scratch in bn_act_bwd layout
        self.dx = None
        self.version = -1

    def pre_reduced(self, dout):
        d, sums = self.dx, self.sums
        self.bn = self.sums = self.dx = None
        if d is None or dout.data_ptr() != d.data_ptr() or dout.shape != d.shape or dout._version != self.version:
            return None
        return sums


class _ResidualBlock(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cfg, *params):
        """cfg: tuple of per-layer (stride, pad, dil, eps, momentum) for the L main convs [+ downsample last];
        params: per layer (weight, gamma, beta, running_mean, running_var), downsample (if any) last, then the SE's
        (fc1 weight, fc1 bias, fc2 weight, fc2 bias) if ``cfg["has_se"]``."""
        n_main, has_ds = cfg["n_main"], cfg["has_ds"]
        layers = [params[5 * i: 5 * i + 5] for i in range(n_main + (1 if has_ds else 0))]
        se = params[5 * len(layers):] if cfg["has_se"] else None
        se_saved = None
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
            groups = cfg["groups"][i]
            wb = weight_bf16(w, groups=groups)
            if groups > 1:      # this step's block-diagonal operand (grouped conv), kept for the data gradient
                wb = native.expand_grouped_weight(wb, w.shape[2] * w.shape[3], groups)
            y, stats = native.conv_fwd(h, wb, (w.shape[2], w.shape[3]), st, pad, dil, stats=True, cout=w.shape[0],
                                       groups=groups)
            last = i == n_main - 1
            if last:      # residual layer: backward masks with 1 bit per element instead of re-reading the block output
                z, save, zmask = native.bn_act_fwd(y, stats, g, b, rm, rv, eps, mom, True, identity, True, want_mask=True)
                cfg["bn3_out"].bn = (y, save, g, b, zmask)
            else:
                z, save = native.bn_act_fwd(y, stats, g, b, rm, rv, eps, mom, True, None, True)
                if se is not None and i == n_main - 2:
                    z, se_saved = _se_fwd(z, *se)
            saved += [h, y, save]
            wbs.append(wb)
            h = z
        ctx.cfg = cfg
        ctx.layers = layers
        ctx.wbs = wbs
        ctx.ds_pack = ds_pack if has_ds else None
        ctx.se = (se, se_saved) if se is not None else None
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
        pre = cfg["bn3_out"].pre_reduced(dout)          # block-output BN sums taken by the next block's dgrad, if any
        for i in range(n_main - 1, -1, -1):
            w, g, b, _, _ = layers[i]
            st, pad, dil, _, _ = cfg["layers"][i]
            h_in, y, save = saved[3 * i], saved[3 * i + 1], saved[3 * i + 2]
            kernel = (w.shape[2], w.shape[3])
            groups = cfg["groups"][i]
            last = i == n_main - 1
            gg = grad_buffer(g) if g.requires_grad else None
            bg = grad_buffer(b) if b.requires_grad else None
            z = None if last else saved[3 * (i + 1)]           # this layer's output = next layer's input (unused: the
            #                                                    mask is recomputed from y; last layer: bit mask)
            # identity shortcut + a dgrad that can add in its epilogue: the shortcut gradient dout * (out > 0) is
            # formed there from dout and the bit mask, so the BN-backward kernel need not write (and dgrad re-read) it
            gate = last and not has_ds and need_dx and cfg["groups"][0] == 1 and native.dgrad_supports_add(
                (layers[0][0].shape[2], layers[0][0].shape[3]), cfg["layers"][0][0])
            dy, dr, _ = native.bn_act_bwd(d, z, y, save, g, True, last and not gate, gg, bg, beta=b, had_residual=last,
                                          zmask=zmask if last else None, pre_reduced=pre)
            if gate:
                gated_add = (dout, zmask)
            if last:
                dres = dr
            pre = None
            if i > 0:
                # where it pays (1x1 dgrads), the dgrad that produces d_{i-1} also reduces dbeta / dgamma of BN_{i-1}
                # in its epilogue (it holds the gradient tile anyway and only has to read the y tile, which it fetches
                # while its MMAs run): BN_{i-1}'s backward is then one pass over (d_{i-1}, y) instead of two
                gp, bp = layers[i - 1][1], layers[i - 1][2]
                se_here = ctx.se is not None and i == n_main - 1     # d is then the gradient at the SE output
                fuse = groups == 1 and not se_here and native.dgrad_fuses_bn_reduce(kernel, st, pad)
                pre = native.zeros_f32((2, h_in.shape[1]), h_in.device) if fuse else None
                d = native.conv_dgrad(dy, ctx.wbs[i], h_in.shape, kernel, st, pad, dil,
                                      bn_reduce=(saved[3 * (i - 1) + 1], gp, bp, saved[3 * (i - 1) + 2], pre)
                                      if fuse else None, groups=groups)
                if se_here:
                    d = _se_bwd(d, ctx.se[1], *ctx.se[0])
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
                # x is the previous block's output: where this dgrad can, it also takes that block's BN3 sums
                prev = cfg["bn3_in"]
                bnr = None
                if prev is not None and prev.bn is not None and groups == 1 and \
                        native.dgrad_fuses_bn_reduce(kernel, st, pad):
                    py, psave, pg, pb, pmask = prev.bn
                    prev.sums = native.zeros_f32((2, x.shape[1]), x.device)
                    bnr = (py, pg, pb, psave, prev.sums, pmask)
                if gated_add is not None:
                    dx = native.conv_dgrad(dy, ctx.wbs[0], x.shape, kernel, st, pad, dil, add=gated_add[0],
                                           add_mask=gated_add[1], bn_reduce=bnr)
                elif groups == 1 and native.dgrad_supports_add(kernel, st):
                    dx = native.conv_dgrad(dy, ctx.wbs[0], x.shape, kernel, st, pad, dil, add=add, bn_reduce=bnr)
                else:
                    bnr = None
                    dx = native.add(native.conv_dgrad(dy, ctx.wbs[0], x.shape, kernel, st, pad, dil, groups=groups),
                                    add)
                if bnr is not None:
                    prev.dx, prev.version = dx, dx._version
            if w.requires_grad:
                gw = grad_buffer(w)
                run_wgrad(w, lambda h_in=h_in, dy=dy, gw=gw, kernel=kernel, st=st, pad=pad, dil=dil, groups=groups:
                          native.conv_wgrad(h_in, dy, gw, kernel, st, pad, dil, groups=groups), h_in, dy)
            for p in (g, b, w):
                if p.requires_grad:
                    notify_ready(p)
        if not need_dx and has_ds and any(p.requires_grad for p in layers[n_main][:3]):
            # block input needs no gradient but (some of) the downsample parameters still do
            wd, gd, bd, _, _ = layers[n_main]
            std, padd, dild, _, _ = cfg["layers"][n_main]
            yd, save_d, wbd = ctx.ds_pack
            dyd, _, _ = native.bn_act_bwd(dres, yd, yd, save_d, gd, False, False,
                                          grad_buffer(gd) if gd.requires_grad else None,
                                          grad_buffer(bd) if bd.requires_grad else None)
            if wd.requires_grad:
                native.conv_wgrad(x, dyd, grad_buffer(wd), (wd.shape[2], wd.shape[3]), std, padd, dild)
            for p in (gd, bd, wd):
                if p.requires_grad:
                    notify_ready(p)
        return (dx, None) + (None,) * (5 * len(layers) + (4 if ctx.se is not None else 0))


def residual_block_supported(x: torch.Tensor, convs: Sequence, bns: Sequence, downsample, se=None) -> bool:
    from .functional import use_native

    if se is not None and (len(convs) < 2 or se.fc1.weight.shape[1] != convs[-2].out_channels):
        return False
    if not use_native(x) or not torch.is_grad_enabled():
        return False
    mods = list(zip(convs, bns)) + ([tuple(downsample)] if downsample is not None else [])
    cin = x.shape[1]
    for conv, bn in mods:
        if not bn.training:
            return False
        if not native.supports_conv(conv.in_channels, conv.out_channels) or not native.bn_supported(conv.out_channels):
            return False
        groups = getattr(conv, "groups", 1)
        if groups > 1 and (not native.grouped_conv_native(conv.in_channels, conv.out_channels, groups) or
                           (downsample is not None and conv is downsample[0])):     # main-path convs only
            return False
        if conv.in_channels <= 4 or not conv.weight.is_contiguous(memory_format=CL) and conv.weight.dim() == 4 and \
                conv.weight.shape[2] * conv.weight.shape[3] > 1:
            return False
    return cin % 8 == 0


def residual_block(x: torch.Tensor, convs: Sequence, bns: Sequence, downsample=None, se=None) -> torch.Tensor:
    """convs/bns: the main-path layer containers (``models.layers.Conv2d`` / ``BatchNorm2d``) in order;
    downsample: optional (conv, bn) pair of the projection shortcut; se: optional squeeze-excitation with ``fc1`` /
    ``fc2`` 1x1 convs (with biases), a ReLU inner activation and a sigmoid gate, applied to the input of the last conv
    (torchvision's RegNetY ``SqueezeExcitation``)."""
    mods = list(zip(convs, bns)) + ([tuple(downsample)] if downsample is not None else [])
    # a block output carries its BN3 handoff; the first block to consume it takes it (a second consumer finds none)
    prev = x.__dict__.pop("_ddl_bn3", None)
    cfg = {"n_main": len(convs), "has_ds": downsample is not None,
           "layers": [(c.stride, c.padding, c.dilation, b.eps, b.momentum) for c, b in mods],
           "groups": [getattr(c, "groups", 1) for c, _ in mods], "has_se": se is not None,
           "bn3_in": prev, "bn3_out": _Bn3Handoff()}
    params = []
    for c, b in mods:
        params += [c.weight, b.weight, b.bias, b.running_mean, b.running_var]
    if se is not None:
        params += [se.fc1.weight, se.fc1.bias, se.fc2.weight, se.fc2.bias]
    out = _ResidualBlock.apply(x, cfg, *params)
    out._ddl_bn3 = cfg["bn3_out"]
    return out
