"""GoogLeNet's Inception module (torchvision's ``Inception``) as ONE autograd node, and the ops of its auxiliary heads.

Widths: c1 (branch1), c2r / c2 (branch2's 1x1 reduction and 3x3), c3r / c3 (branch3's reduction and 3x3, torchvision's
"5x5" branch, which uses a 3x3 kernel), c4 (the pool projection); M = N * H * W rows.

    forward   p = maxpool3x3/s1/p1(x)                                   (arg-max codes saved)
              R = x . [W1; W2r; W3r]^T               [M, c1 + c2r + c3r]   ONE 1x1 GEMM, BN sums in its epilogue
              out[:, :c1] = relu(BN1(R1)), t2 = relu(BN2r(R2)), t3 = relu(BN3r(R3))          one bn_seg_fwd
              y2 = conv3x3(t2), y3 = conv3x3(t3), y4 = conv1x1(p)                           BN sums in the epilogues
              out[:, c1:] = relu(BN2(y2)), relu(BN3(y3)), relu(BN4(y4))                     one bn_seg_fwd
    backward  dout's four segments -> dR[:, :c1], dy2, dy3, dy4                             one bn_seg_bwd
              dt2, dt3 = dgrad3x3(dy2), dgrad3x3(dy3); dp = dgrad1x1(dy4)
              dt2, dt3 -> dR[:, c1:]                                                         one bn_seg_bwd
              dx = dgrad1x1(dR, [W1; W2r; W3r]) + maxpool_bwd(dp)                            ONE store of dx
              weight gradients on the side stream (``run_wgrad``); the merged 1x1 gradient is folded into the three
              torchvision-shaped ``.grad`` slots in one launch; ``notify_ready`` last for every parameter

The segmented BN kernels (csrc/ops/inception.cu) read and write strided channel slices, so ``out`` is written once in
place: there is no concat or split copy, and autograd never sums two gradients of x.  The conv kernels only see
contiguous tensors.  The stacked bf16 weight is built from the weight arena views in one launch every step, so a
captured CUDA graph rebuilds it on replay.  The node stays bf16 in fp8 sessions: its reductions (K = 480, 832, ...) do
not all meet the fp8 path's multiple-of-128 rule, and one node keeps one precision.

:func:`inception_module_composite` (torch ops) is the CPU path and the float64 oracle of the tests.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn.functional as F

from . import fp8, native
from .functional import CL, grad_buffer, notify_ready, run_wgrad, use_native, weight_bf16

_B1, _B2R, _B2, _B3R, _B3, _B4 = range(6)


def _bn_args(bn) -> tuple:
    return (bn.weight, bn.bias, bn.running_mean, bn.running_var)


class _Plan:
    """A module's widths (cin, c1, c2r, c2, c3r, c3, c4) and its BN mode."""

    def __init__(self, widths, training: bool):
        self.widths, self.training = tuple(widths), training


class _Inception(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan, save, eps_mom, *ps):
        """ps: per layer (weight, gamma, beta, running_mean, running_var) of branch1, branch2's 1x1 and 3x3, branch3's
        1x1 and 3x3, branch4's 1x1."""
        with fp8.bf16_only():
            return _Inception._forward(ctx, x, plan, save, eps_mom, ps)

    @staticmethod
    def _forward(ctx, x, plan, save, eps_mom, ps):
        cin, c1, c2r, c2, c3r, c3, c4 = plan.widths
        training = plan.training
        L = [ps[i:i + 5] for i in range(0, len(ps), 5)]
        N, _, H, W = x.shape
        dev = x.device
        ctot = c1 + c2r + c3r
        # [W1; W2r; W3r] from the bf16 arena views in one launch
        wcat = torch.empty((ctot, cin), dtype=torch.bfloat16, device=dev)
        native.pad_cols([(weight_bf16(L[i][0]), c, cin, wcat[o:o + c])
                         for i, c, o in ((_B1, c1, 0), (_B2R, c2r, c1), (_B3R, c3r, c1 + c2r))])
        wb2, wb3, wb4 = weight_bf16(L[_B2][0]), weight_bf16(L[_B3][0]), weight_bf16(L[_B4][0])

        def conv(h, wb, k, cout):
            if training:
                return native.conv_fwd(h, wb, (k, k), 1, k // 2, stats=True, cout=cout)
            return native.conv_fwd(h, wb, (k, k), 1, k // 2, cout=cout), None

        saves = [torch.empty((2, L[i][1].numel()), dtype=torch.float32, device=dev) if training else None
                 for i in range(6)]

        def seg(i, src, scol, dst, dcol, st, soff):
            g, b, rm, rv = L[i][1:5]
            c = g.numel()
            d = dict(x=(src, scol), z=(dst, dcol), c=c, gamma=g, beta=b, running_mean=rm, running_var=rv,
                     eps=eps_mom[i][0], momentum=eps_mom[i][1])
            if training:
                d.update(sum=st[0, soff:soff + c], sumsq=st[1, soff:soff + c], mean=saves[i][0], invstd=saves[i][1])
            return d

        p, arg = native.maxpool_fwd(x, 3, 1, 1, True)
        R, stR = conv(x, wcat, 1, ctot)
        out = native.empty_act(N, c1 + c2 + c3 + c4, H, W, dev)
        t2, t3 = native.empty_act(N, c2r, H, W, dev), native.empty_act(N, c3r, H, W, dev)
        native.bn_seg_fwd([seg(_B1, R, 0, out, 0, stR, 0), seg(_B2R, R, c1, t2, 0, stR, c1),
                           seg(_B3R, R, c1 + c2r, t3, 0, stR, c1 + c2r)], training)
        y2, st2 = conv(t2, wb2, 3, c2)
        y3, st3 = conv(t3, wb3, 3, c3)
        y4, st4 = conv(p, wb4, 1, c4)
        native.bn_seg_fwd([seg(_B2, y2, 0, out, c1, st2, 0), seg(_B3, y3, 0, out, c1 + c2, st3, 0),
                           seg(_B4, y4, 0, out, c1 + c2 + c3, st4, 0)], training)
        ctx.plan, ctx.layers = plan, L
        ctx.saved_ok = save
        if save:
            ctx.wbs = (wcat, wb2, wb3, wb4)        # this step's stacked copy / views of the bf16 weight arena
            ctx.save_for_backward(x, p, arg, R, t2, t3, y2, y3, y4, *saves)
        return out

    @staticmethod
    def backward(ctx, dout):
        if not ctx.saved_ok:
            raise RuntimeError("inception_module: no backward through a module run with its BatchNorms in eval mode "
                               "(the native node, like conv_bn_act's, saves nothing in eval); train the module, or "
                               "run eval under torch.no_grad()")
        with fp8.bf16_only():
            dx = _Inception._backward(ctx, dout)
        return (dx, None, None, None) + (None,) * 30

    @staticmethod
    def _backward(ctx, dout):
        cin, c1, c2r, c2, c3r, c3, c4 = ctx.plan.widths
        L = ctx.layers
        x, p, arg, R, t2, t3, y2, y3, y4, *saves = ctx.saved_tensors
        wcat, wb2, wb3, wb4 = ctx.wbs
        if not dout.is_contiguous(memory_format=CL):
            dout = dout.contiguous(memory_format=CL)
        N, _, H, W = x.shape
        dev = x.device
        ctot = c1 + c2r + c3r

        def seg(i, dz, dzcol, src, scol, dst, dcol):
            g, b = L[i][1], L[i][2]
            return dict(dz=(dz, dzcol), x=(src, scol), dx=(dst, dcol), c=g.numel(), gamma=g, beta=b,
                        mean=saves[i][0], invstd=saves[i][1],
                        gamma_grad=grad_buffer(g) if g.requires_grad else None,
                        beta_grad=grad_buffer(b) if b.requires_grad else None)

        def wgrad(i, h, dy, k):
            w = L[i][0]
            if w.requires_grad:
                gw = grad_buffer(w)
                run_wgrad(w, lambda: native.conv_wgrad(h, dy, gw, (k, k), 1, k // 2), h, dy)

        dR = native.empty_act(N, ctot, H, W, dev)
        dy2, dy3, dy4 = (native.empty_act(N, c, H, W, dev) for c in (c2, c3, c4))
        native.bn_seg_bwd([seg(_B1, dout, 0, R, 0, dR, 0), seg(_B2, dout, c1, y2, 0, dy2, 0),
                           seg(_B3, dout, c1 + c2, y3, 0, dy3, 0), seg(_B4, dout, c1 + c2 + c3, y4, 0, dy4, 0)])
        dt2 = native.conv_dgrad(dy2, wb2, t2.shape, (3, 3), 1, 1)
        wgrad(_B2, t2, dy2, 3)
        dt3 = native.conv_dgrad(dy3, wb3, t3.shape, (3, 3), 1, 1)
        wgrad(_B3, t3, dy3, 3)
        native.bn_seg_bwd([seg(_B2R, dt2, 0, R, c1, dR, c1), seg(_B3R, dt3, 0, R, c1 + c2r, dR, c1 + c2r)])
        wgrad(_B4, p, dy4, 1)
        dx = None
        if ctx.needs_input_grad[0]:
            dp = native.conv_dgrad(dy4, wb4, p.shape, (1, 1), 1, 0)
            dx = native.conv_dgrad(dR, wcat, x.shape, (1, 1), 1, 0, add=native.maxpool_bwd(dp, arg, x.shape, 3, 1, 1))
        merged = [(i, c, o) for i, c, o in ((_B1, c1, 0), (_B2R, c2r, c1), (_B3R, c3r, c1 + c2r))
                  if L[i][0].requires_grad]
        if merged:
            gw = torch.zeros((ctot, cin), dtype=torch.float32, device=dev)
            folds = [(gw[o:o + c], grad_buffer(L[i][0]), c) for i, c, o in merged]

            def merged_wgrad():
                native.conv_wgrad(x, dR, gw, (1, 1), 1, 0)
                native.fold_cols(folds)

            run_wgrad(L[merged[0][0]][0], merged_wgrad, x, dR, gw)
        for lay in L:             # LAST, as in functional._ConvBnAct
            for t in lay[:3]:
                if t.requires_grad:
                    notify_ready(t)
        return dx


def inception_native(x) -> bool:
    """Whether an input runs on the native node: an NHWC bf16 CUDA activation under the native implementation."""
    return use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)


def inception_module(x, convs: Sequence):
    """torchvision's ``Inception`` on ``convs`` = (branch1, branch2[0], branch2[1], branch3[0], branch3[1],
    branch4[1]): ``BasicConv2d`` holders with ``.conv`` / ``.bn`` (``models.inception``).  The native node on NHWC bf16
    CUDA activations whose widths are multiples of 8, the composite elsewhere."""
    bns = [m.bn for m in convs]
    training = bns[0].training
    if any(b.training != training for b in bns):
        raise ValueError("inception_module: all BatchNorms of a module must be in the same mode")
    ws = [m.conv.weight for m in convs]
    widths = (ws[0].shape[1], ws[0].shape[0], ws[1].shape[0], ws[2].shape[0], ws[3].shape[0], ws[4].shape[0],
              ws[5].shape[0])
    if not inception_native(x) or any(c % 8 for c in widths):
        layers = [(w, _bn_args(b) + (b.eps, b.momentum)) for w, b in zip(ws, bns)]
        return inception_module_composite(x, layers, training)
    if x.shape[1] != widths[0]:
        raise ValueError(f"inception_module: the input has {x.shape[1]} channels, the module takes {widths[0]}")
    ps = [t for w, b in zip(ws, bns) for t in (w,) + _bn_args(b)]
    save = training and torch.is_grad_enabled() and (x.requires_grad or any(t.requires_grad for t in ps))
    eps_mom = tuple((b.eps, b.momentum) for b in bns)
    return _Inception.apply(x, _Plan(widths, training), save, eps_mom, *ps)


def inception_module_composite(x, layers, training=True, relus=None) -> torch.Tensor:
    """torchvision's ``Inception`` in torch ops.  ``layers`` = six (weight, bn) pairs in the order of
    :func:`inception_module`, bn = (gamma, beta, running_mean, running_var, eps, momentum).  On CPU in the weights'
    dtype, on CUDA in the activations' dtype with the BNs in fp32.  In float64 it is the oracle of the tests.
    ``relus``: six callables in place of the layers' ReLUs (the tests' float64 twin passes ReLUs that follow the tested
    implementation's side where the input is within bf16 rounding of zero); default ``F.relu``."""
    dt = x.dtype if x.is_cuda else layers[0][0].dtype
    x = x.to(dt)
    acts = relus if relus is not None else (F.relu,) * 6

    def cbr(h, i):
        w, (g, b, rm, rv, eps, mom) = layers[i]
        y = F.conv2d(h, w.to(dt), None, 1, w.shape[2] // 2)
        yb = y.float() if y.dtype in (torch.bfloat16, torch.float16) else y
        return acts[i](F.batch_norm(yb, rm, rv, g, b, training, mom, eps).to(y.dtype))

    out = torch.cat([cbr(x, _B1), cbr(cbr(x, _B2R), _B2), cbr(cbr(x, _B3R), _B3),
                     cbr(F.max_pool2d(x, 3, 1, 1, ceil_mode=True), _B4)], 1)
    return out.contiguous(memory_format=CL) if out.is_cuda else out


# ------------------------------------------------------------------------------------------------
# the auxiliary head: adaptive average pooling and the NCHW-order flatten
# ------------------------------------------------------------------------------------------------
class _AdaptiveAvgPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, out_hw):
        ctx.shape = x.shape
        return native.adaptive_avgpool_fwd(x, out_hw)

    @staticmethod
    def backward(ctx, dy):
        if not dy.is_contiguous(memory_format=CL):
            dy = dy.contiguous(memory_format=CL)
        return native.adaptive_avgpool_bwd(dy, ctx.shape), None


def adaptive_avg_pool2d(x, output_size):
    """``F.adaptive_avg_pool2d`` with torch's (overlapping) windows; native on NHWC bf16 activations whose channel
    count is a multiple of 8."""
    out_hw = (output_size, output_size) if isinstance(output_size, int) else tuple(output_size)
    if inception_native(x) and x.shape[1] % 8 == 0 and out_hw[0] <= x.shape[2] and out_hw[1] <= x.shape[3]:
        return _AdaptiveAvgPool.apply(x, out_hw)
    return F.adaptive_avg_pool2d(x, out_hw)


class _FlattenNCHW(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        n, c, h, w = x.shape
        ctx.shape = x.shape
        return native.transpose_rows(x, h * w, c)

    @staticmethod
    def backward(ctx, dy):
        n, c, h, w = ctx.shape
        dx = native.transpose_rows(dy.contiguous(), c, h * w)         # [N, HW * C]: NHWC memory
        return dx.view(n, h, w, c).permute(0, 3, 1, 2)


def flatten_nchw(x):
    """``torch.flatten(x, 1)`` of an activation [N, C, H, W], in torchvision's NCHW order (index c * H * W + h * W + w)
    whatever its memory layout; native (one permutation launch each way) on NHWC bf16 activations with C and H * W
    multiples of 8."""
    if inception_native(x) and x.shape[1] % 8 == 0 and (x.shape[2] * x.shape[3]) % 8 == 0:
        return _FlattenNCHW.apply(x)
    return torch.flatten(x, 1)
