"""ShuffleNetV2's unit (torchvision's ``InvertedResidual``) as ONE autograd node.

    stride 1   x1, x2 = x.chunk(2);  b = relu(BN3(conv1x1(BN2(dw3x3(relu(BN1(conv1x1(x2))))))));
               s = shuffle(cat(x1, b))
    stride 2   a = relu(BNp(conv1x1(BNd(dw3x3_s2(x)))));  b as above on x with a stride-2 depthwise;
               s = shuffle(cat(a, b))

with shuffle(.)[2i] = first half [i], [2i+1] = second half [i].  The branches run on the conv (1x1 GEMM), depthwise 3x3
and BN kernels; the last BN of each branch, the concat and the shuffle are one pass of ``native.shuffle_fwd``
(csrc/ops/shufflenet.cu), which writes s either whole or as its two channel halves lo = s[:, :C/2], hi = s[:, C/2:].
A unit hands the next one (lo, hi): a stride-1 unit reads lo as its pass-through and hi as its branch input, so no
channel slice is ever copied.  The last unit of a stage writes s whole, because a stride-2 unit or ``conv5`` reads all
of it.  Backward: ``native.shuffle_bwd`` de-interleaves the output gradient in the BN-backward passes of the branch
half (halves) and copies the pass-through gradient; the stride-2 input gradient is branch1's depthwise data gradient
added in the store of branch2's 1x1 data gradient (``conv_dgrad(..., add=)``).

Padded layout (decided here alone): every activation this node stores, lo / hi / s included, holds its real channels
first and zero channels up to p(c) = c rounded up to 8, so the widths of x1.0 (58, 116) and x2.0 (122, 244) run on the
kernels, which take multiples of 8.  Such a unit pads its operands in one launch every step, from the bf16 weight arena
views and the fp32 parameters: 1x1 weights to [p(Cout), p(Cin)], depthwise weights to [p(C), 9], the inner BNs'
gamma / beta (zero in the pad) and running statistics to p(c).  Its weight and BN parameter gradients go to one padded
fp32 scratch and are folded into torchvision-shaped ``.grad`` slots in one launch; the inner BNs' running statistics
are copied back in one launch after a training forward.  The branch's last BN (and branch1's) runs in the shuffle
kernels on the real channels, with the unpadded parameters.  Units whose widths are all multiples of 8 take no pad or
fold launch.  The node stays bf16: none of ShuffleNetV2's convolutions has the multiple-of-128 widths of the fp8 path.

:func:`shuffle_unit_composite` (torch ops, torchvision's channel order, no padding) is the CPU path and the float64
oracle of the tests.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn.functional as F

from . import native
from .functional import CL, grad_buffer, notify_ready, run_wgrad, use_native, weight_bf16


def _p8(c: int) -> int:
    return (c + 7) // 8 * 8


def _bn_args(bn) -> tuple:
    return (bn.weight, bn.bias, bn.running_mean, bn.running_var)


class _Plan:
    """A unit's stride, real input and branch widths, whether any of them needs the padded layout, and its BN mode
    (``training``, set by :func:`shuffle_unit`)."""

    def __init__(self, stride: int, cin: int, bf: int):
        self.stride, self.cin, self.bf = stride, cin, bf
        self.pad = cin % 8 != 0 or bf % 8 != 0


class _ShuffleUnit(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x0, x1, plan, whole, save, eps_mom, *ps):
        """x0, x1: (lo, hi) of a stride-1 unit, or (x, None) of a stride-2 one.  ps: per layer (weight, gamma, beta,
        running_mean, running_var): branch1's depthwise and 1x1 (stride 2), then branch2's 1x1, depthwise and 1x1."""
        training = plan.training
        layers = [ps[i:i + 5] for i in range(0, len(ps), 5)]
        two = plan.stride == 2
        kinds = (["dw", "1x1"] if two else []) + ["1x1", "dw", "1x1"]
        bf, cin = plan.bf, plan.cin
        pb, pc = _p8(bf), _p8(cin)
        # bf16 operands: views of the weight arena, padded in one launch when a width is not a multiple of 8
        wbs = []
        for kind, lay in zip(kinds, layers):
            w = lay[0]
            wbs.append(weight_bf16(w, groups=w.shape[0]) if kind == "dw" else weight_bf16(w))
        inner = [i for i in range(len(layers)) if i not in ((1, 4) if two else (2,))]     # BNs before the shuffle
        vecs = {i: list(layers[i][1:5]) for i in inner}
        if plan.pad:
            shapes = []
            for i, (kind, w) in enumerate(zip(kinds, wbs)):
                rows = pc if (two and i == 0) else pb
                shapes.append((w, rows, 9 if kind == "dw" else (pc if w.shape[1] == cin else pb)))
            for i in inner:
                c = pc if (two and i == 0) else pb
                shapes += [(v, 1, c) for v in vecs[i]]
            out = native.pad_cols(shapes)
            wbs = out[:len(wbs)]
            k = len(wbs)
            for i in inner:
                vecs[i] = [t.view(-1) for t in out[k:k + 4]]
                k += 4

        def conv(h, i, stride=1):
            if kinds[i] == "dw":
                return native.dwconv_fwd(h, wbs[i], stride, stats=training) if training \
                    else (native.dwconv_fwd(h, wbs[i], stride), None)
            return native.conv_fwd(h, wbs[i], (1, 1), 1, 0, stats=training, cout=wbs[i].shape[0]) if training \
                else (native.conv_fwd(h, wbs[i], (1, 1), 1, 0, cout=wbs[i].shape[0]), None)

        def bn(y, st, i, relu):
            g, b, rm, rv = vecs[i]
            return native.bn_act_fwd(y, st, g, b, rm, rv, eps_mom[i][0], eps_mom[i][1], relu, None, training)

        def last_bn(st, i, save_t):
            g, b, rm, rv = layers[i][1:5]
            d = dict(gamma=g, beta=b, running_mean=rm, running_var=rv, eps=eps_mom[i][0], momentum=eps_mom[i][1])
            if training:
                d.update(sum=st[0], sumsq=st[1], mean=save_t[0], invstd=save_t[1])
            return d

        saved = []
        bn_a = a = None
        if two:
            x = x0
            yd, std = conv(x, 0, 2)
            hd, svd = bn(yd, std, 0, False)
            a, sta = conv(hd, 1)
            sva = torch.empty((2, bf), dtype=torch.float32, device=x.device)
            bn_a = last_bn(sta, 1, sva)
            saved += [x, yd, svd, hd, a, sva]
            xb, o = x, 2
        else:
            xb, o = x1, 0
            a = x0
        y1, st1 = conv(xb, o)
        h1, sv1 = bn(y1, st1, o, True)
        y2, st2 = conv(h1, o + 1, plan.stride)
        h2, sv2 = bn(y2, st2, o + 1, False)
        y3, st3 = conv(h2, o + 2)
        sv3 = torch.empty((2, bf), dtype=torch.float32, device=y3.device)
        out = native.shuffle_fwd(a, y3, bf, not whole, training, last_bn(st3, o + 2, sv3), bn_a)
        if training and plan.pad:         # the inner BNs updated their padded running statistics: copy them back
            native.fold_cols([(vecs[i][j], layers[i][j + 1], 1) for i in inner for j in (2, 3)], add=False)
        saved += [xb, y1, sv1, h1, y2, sv2, h2, y3, sv3]
        ctx.plan, ctx.kinds, ctx.whole, ctx.inner = plan, kinds, whole, inner
        ctx.layers = layers
        if save:
            ctx.wbs, ctx.vecs = wbs, vecs           # views of the bf16 weight arena / this step's padded copies
            ctx.save_for_backward(*saved)
        ctx.saved_ok = save
        return out

    @staticmethod
    def backward(ctx, *grads):
        if not ctx.saved_ok:
            raise RuntimeError("shuffle_unit: no backward through a unit run with its BatchNorms in eval mode "
                               "(the native node, like conv_bn_act's, saves nothing in eval); train the unit, or "
                               "run eval under torch.no_grad()")
        plan, kinds, layers, inner = ctx.plan, ctx.kinds, ctx.layers, ctx.inner
        two, bf, cin = plan.stride == 2, plan.bf, plan.cin
        pb, pc = _p8(bf), _p8(cin)
        grads = [g if g.is_contiguous(memory_format=CL) else g.contiguous(memory_format=CL) for g in grads]
        ds = grads[0] if ctx.whole else (grads[0], grads[1])
        st = list(ctx.saved_tensors)
        wbs, vecs = ctx.wbs, ctx.vecs
        # gradient targets: the .grad slots, or views of one padded fp32 scratch folded into them at the end
        targets, folds = {}, []
        if plan.pad:
            sizes = []
            for i, kind in enumerate(kinds):
                sizes.append(wbs[i].numel())
                if i in inner:
                    sizes += [pc if (two and i == 0) else pb] * 2
            scratch = torch.zeros(sum(sizes), dtype=torch.float32, device=wbs[0].device)
            parts = iter(scratch.split(sizes))
            for i, kind in enumerate(kinds):
                w = layers[i][0]
                wv = next(parts).view(wbs[i].shape)
                targets[(i, 0)] = wv.view(wbs[i].shape[0], 1, 3, 3) if kind == "dw" else wv.view(*wbs[i].shape, 1, 1)
                if w.requires_grad:
                    folds.append((wv, grad_buffer(w), w.shape[0]))
                if i in inner:
                    for j in (1, 2):
                        v = next(parts)
                        targets[(i, j)] = v
                        if layers[i][j].requires_grad:
                            folds.append((v.view(1, -1), grad_buffer(layers[i][j]), 1))

        def target(i, j):
            p = layers[i][j]
            if not p.requires_grad:
                return None
            return targets[(i, j)] if plan.pad and (i, j) in targets else grad_buffer(p)

        def last_bn(i, save_t):
            g, b = layers[i][1], layers[i][2]
            scr = native.zeros_f32((2, bf), save_t.device)
            return dict(gamma=g, beta=b, mean=save_t[0], invstd=save_t[1], dgamma=scr[0], dbeta=scr[1],
                        gamma_grad=grad_buffer(g) if g.requires_grad else None,
                        beta_grad=grad_buffer(b) if b.requires_grad else None)

        def bn_bwd(dz, y, save_t, i, relu):
            g, b = vecs[i][0], vecs[i][1]
            dy, _, _ = native.bn_act_bwd(dz, None, y, save_t, g, relu, False, target(i, 1), target(i, 2), beta=b,
                                         had_residual=False)
            return dy

        def wgrad(i, h, dy, stride=1):
            if not layers[i][0].requires_grad:
                return
            t = target(i, 0)
            if kinds[i] == "dw":
                run_wgrad(layers[i][0], lambda: native.dwconv_wgrad(h, dy, t, stride), h, dy)
            else:
                run_wgrad(layers[i][0], lambda: native.conv_wgrad(h, dy, t, (1, 1), 1, 0), h, dy)

        xb, y1, sv1, h1, y2, sv2, h2, y3, sv3 = st[-9:]
        o = 2 if two else 0
        dx1 = None
        if two:
            x, yd, svd, hd, a, sva = st[:6]
            da, dy3 = native.shuffle_bwd(ds, y3, bf, last_bn(o + 2, sv3), a=a, bn_a=last_bn(1, sva))
            dhd = native.conv_dgrad(da, wbs[1], hd.shape, (1, 1), 1, 0)
            wgrad(1, hd, da)
            dyd = bn_bwd(dhd, yd, svd, 0, False)
            if ctx.needs_input_grad[0]:
                dx1 = native.dwconv_dgrad(dyd, wbs[0], x.shape, 2)
            wgrad(0, x, dyd, 2)
            dpass = None
        else:
            dpass, dy3 = native.shuffle_bwd(ds, y3, bf, last_bn(o + 2, sv3))
        dh2 = native.conv_dgrad(dy3, wbs[o + 2], h2.shape, (1, 1), 1, 0)
        wgrad(o + 2, h2, dy3)
        dy2 = bn_bwd(dh2, y2, sv2, o + 1, False)
        dh1 = native.dwconv_dgrad(dy2, wbs[o + 1], h1.shape, plan.stride)
        wgrad(o + 1, h1, dy2, plan.stride)
        dy1 = bn_bwd(dh1, y1, sv1, o, True)
        need_xb = ctx.needs_input_grad[0] if two else ctx.needs_input_grad[1]
        dxb = native.conv_dgrad(dy1, wbs[o], xb.shape, (1, 1), 1, 0, add=dx1) if need_xb else None
        wgrad(o, xb, dy1)
        params = [p for lay in layers for p in lay[:3] if p.requires_grad]
        if folds:
            run_wgrad(params[0], lambda: native.fold_cols(folds), scratch)
        for p in params:          # LAST, as in functional._ConvBnAct
            notify_ready(p)
        if two:
            return (dxb, None, None, None, None, None) + (None,) * len(layers) * 5
        return (dpass if ctx.needs_input_grad[0] else None, dxb, None, None, None, None) + (None,) * len(layers) * 5


def shuffle_unit_native(x) -> bool:
    """Whether a unit input runs on the native node: a (lo, hi) pair from the previous node, or an NHWC bf16 CUDA tensor
    under the native implementation."""
    if isinstance(x, tuple):
        return True
    return use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)


def shuffle_unit(x, branch1: Optional[Sequence], branch2: Sequence, whole_output: bool = True):
    """torchvision's ``InvertedResidual``: ``branch1`` = None (stride 1) or (depthwise conv, BN, 1x1 conv, BN) holders,
    ``branch2`` = (1x1 conv, BN, depthwise conv, BN, 1x1 conv, BN) holders (``models.layers``).  On the native node the
    input is the previous unit's (lo, hi) pair (stride 1) or a whole NHWC bf16 tensor (stride 2, its channels padded to
    a multiple of 8 with zeros), and the output is (lo, hi), or s whole with ``whole_output``.  Elsewhere (CPU, or the
    torch implementation on CUDA) the composite in torchvision's layout: a tensor in, a tensor out."""
    stride = 2 if branch1 is not None else 1
    bns = ([branch1[1], branch1[3]] if branch1 is not None else []) + [branch2[1], branch2[3], branch2[5]]
    convs = ([branch1[0], branch1[2]] if branch1 is not None else []) + [branch2[0], branch2[2], branch2[4]]
    training = bns[0].training
    if any(b.training != training for b in bns):
        raise ValueError("shuffle_unit: all BatchNorms of a unit must be in the same mode")
    if not shuffle_unit_native(x):
        b1 = None if branch1 is None else (convs[0].weight, _bn_args(bns[0]) + (bns[0].eps, bns[0].momentum),
                                           convs[1].weight, _bn_args(bns[1]) + (bns[1].eps, bns[1].momentum))
        o = 0 if branch1 is None else 2
        b2 = tuple(t for i in range(3) for t in (convs[o + i].weight,
                                                   _bn_args(bns[o + i]) + (bns[o + i].eps, bns[o + i].momentum)))
        return shuffle_unit_composite(x, b2, b1, training)
    bf = convs[-1].weight.shape[0]
    cin = convs[0].weight.shape[0] if stride == 2 else bf
    if bf % 2 != 0:
        raise ValueError(f"shuffle_unit: the native node needs an even branch width, got {bf}")
    if stride == 1 and not isinstance(x, tuple):
        raise ValueError("shuffle_unit: a stride-1 unit on the native node takes the previous unit's (lo, hi) pair")
    if stride == 2 and (isinstance(x, tuple) or x.shape[1] != _p8(cin)):
        raise ValueError(f"shuffle_unit: a stride-2 unit takes a whole tensor of {_p8(cin)} channels")
    plan = _Plan(stride, cin, bf)
    plan.training = training
    ps = [t for c, b in zip(convs, bns) for t in (c.weight,) + _bn_args(b)]
    x0, x1 = x if stride == 1 else (x, None)
    inputs = [x0] + ([x1] if x1 is not None else [])
    save = training and torch.is_grad_enabled() and (any(t.requires_grad for t in inputs) or any(
        p.requires_grad for p in ps))
    eps_mom = tuple((b.eps, b.momentum) for b in bns)
    return _ShuffleUnit.apply(x0, x1, plan, whole_output, save, eps_mom, *ps)


def channel_shuffle(x: torch.Tensor, groups: int = 2) -> torch.Tensor:
    n, c, h, w = x.shape
    return x.view(n, groups, c // groups, h, w).transpose(1, 2).reshape(n, c, h, w)


def shuffle_unit_composite(x, branch2, branch1=None, training=True, relus=None) -> torch.Tensor:
    """torchvision's ``InvertedResidual`` in torch ops.  ``branch2`` = (w1, bn1, w_dw, bn2, w3, bn3), ``branch1`` = None
    (stride 1) or (w_dw, bn, w_1x1, bn), each bn = (gamma, beta, running_mean, running_var, eps, momentum); the stride
    is 2 with a branch1.  On CPU in the weights' dtype, on CUDA in the activations' dtype with the BNs in fp32.  In float64
    it is the oracle of the tests.  ``relus``: three callables in place of the ReLUs after branch2's first BN, branch2's
    last BN and branch1's last BN (the tests' float64 twin passes ReLUs that follow the tested implementation's side
    where the input is within bf16 rounding of zero); default ``F.relu``."""
    dt = x.dtype if x.is_cuda else branch2[0].dtype
    x = x.to(dt)
    stride = 2 if branch1 is not None else 1
    r_inner, r_last, r_b1 = relus if relus is not None else (F.relu,) * 3

    def bn(y, p, act=None):
        g, b, rm, rv, eps, mom = p
        yb = y.float() if y.dtype in (torch.bfloat16, torch.float16) else y
        z = F.batch_norm(yb, rm, rv, g, b, training, mom, eps).to(y.dtype)
        return act(z) if act is not None else z

    def dw(h, w, s):
        return F.conv2d(h, w.to(dt), None, s, 1, 1, w.shape[0])

    if branch1 is None:
        a, xb = x.chunk(2, dim=1)
    else:
        a = bn(F.conv2d(bn(dw(x, branch1[0], 2), branch1[1]), branch1[2].to(dt)), branch1[3], r_b1)
        xb = x
    w1, bn1, wd, bn2, w3, bn3 = branch2
    h = bn(F.conv2d(xb, w1.to(dt)), bn1, r_inner)
    h = bn(dw(h, wd, stride), bn2)
    b = bn(F.conv2d(h, w3.to(dt)), bn3, r_last)
    return channel_shuffle(torch.cat((a, b), dim=1), 2)
