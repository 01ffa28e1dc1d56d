"""Differentiable fused ops: native sm_90a kernels on CUDA, plain PyTorch composites on CPU.

Each public function has ONE GPU implementation (the hand-written kernels; there is no
cuDNN/cuBLAS/ATen alternative behind a switch on the flagship path) and a CPU implementation built
from stock torch ops that doubles as the fp32 numerics oracle in tests (``--no-cuda`` mode of the
reference scripts, SURVEY.md section 4).  ``DDL_B200_IMPL=torch`` forces the composite on GPU as a
debugging aid (A/B numerics), never as a fallback: if the native module cannot be loaded on a CUDA
device the call raises.

Gradients of parameters are accumulated by the kernels DIRECTLY into ``param.grad`` (the fp32
bucket arena slot when a fused engine is attached — SURVEY.md K4/K12) and the parameter's
``_ddl_ready`` callback is invoked; autograd only carries activation gradients.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from . import native

CL = torch.channels_last


def use_native(x: torch.Tensor) -> bool:
    if not x.is_cuda:
        return False
    return os.environ.get("DDL_B200_IMPL", "native") != "torch"


# ------------------------------------------------------------------------------------------------
# parameter-side helpers
# ------------------------------------------------------------------------------------------------
def grad_buffer(p: torch.Tensor) -> torch.Tensor:
    """fp32 gradient accumulator with the SAME memory layout as ``p`` (created zeroed on demand)."""
    if p.grad is None:
        p.grad = torch.zeros_like(p, memory_format=torch.preserve_format)
    return p.grad


# ------------------------------------------------------------------------------------------------
# weight-gradient side stream
# ------------------------------------------------------------------------------------------------
# wgrad kernels feed only the optimizer, never the rest of backward.  When a fused engine is attached (it joins this
# stream before it consumes a bucket) they are enqueued on a side stream so they overlap the dgrad -> BN-backward chain
# of the earlier layers: the conv kernels are latency-bound per tile and the BN kernels are HBM-bound, so co-residency
# fills otherwise idle issue slots.  DDL_ASYNC_WGRAD=0 restores single-stream execution.
_WGRAD = {"stream": None, "enabled": os.environ.get("DDL_ASYNC_WGRAD", "1") != "0", "pending": False, "native": False}


def use_native_wgrad_join(on: bool) -> None:
    """The engine's native StepLauncher joins the side stream itself (csrc/runtime/step_launcher.cpp): side-stream work
    is then noted in the native module instead of the Python flag."""
    _WGRAD["native"] = bool(on)


def wgrad_stream() -> Optional["torch.cuda.Stream"]:
    return _WGRAD["stream"]


def wgrad_join(consumer: "torch.cuda.Stream") -> None:
    """Make ``consumer`` wait for the weight-gradient kernels enqueued on the side stream since the last join.
    Skipped when nothing is pending: besides saving an event, that keeps CUDA-graph capture legal (a capturing stream
    must not wait on a stream that has not joined the capture yet)."""
    side = _WGRAD["stream"]
    if _WGRAD["native"]:
        from .. import _ext

        _ext.load().wgrad_join(consumer.cuda_stream)
    elif side is not None and _WGRAD["pending"]:
        consumer.wait_stream(side)
        _WGRAD["pending"] = False


def run_wgrad(param: torch.Tensor, fn, *tensors: torch.Tensor) -> None:
    """Run ``fn()`` (a wgrad launch for ``param``) — on the side stream when the engine will join it."""
    if not _WGRAD["enabled"] or getattr(param, "_ddl_ready", None) is None:
        fn()
        return
    if _WGRAD["stream"] is None:
        _WGRAD["stream"] = torch.cuda.Stream(device=param.device)
    side = _WGRAD["stream"]
    side.wait_stream(torch.cuda.current_stream(param.device))
    with torch.cuda.stream(side):
        fn()
    if _WGRAD["native"]:
        from .. import _ext

        _ext.load().wgrad_note(side.cuda_stream)
    else:
        _WGRAD["pending"] = True
    if not torch.cuda.is_current_stream_capturing():
        for t in tensors:
            t.record_stream(side)


def notify_ready(p: torch.Tensor) -> None:
    cb = getattr(p, "_ddl_ready", None)
    if cb is not None:
        cb()


def weight_bf16(p: torch.Tensor, kernel: Optional[Tuple[int, int]] = None) -> torch.Tensor:
    """bf16 GEMM operand of a parameter.

    With a fused engine attached the copy is a view into the bf16 weight arena that the
    allreduce+SGD kernel refreshes every step (no per-step cast).  Otherwise it is cast on
    demand and cached against the parameter's version counter.  Stem weights (Cin <= 4) are
    re-packed to the padded [Cout, KB*64] matrix.
    """
    stem = p.dim() == 4 and p.shape[1] <= 4
    view = getattr(p, "_ddl_bf16", None)
    if view is not None and not stem:
        return view
    cache = getattr(p, "_ddl_cast_cache", None)
    ver = p._version
    if cache is not None and cache[0] == ver and cache[1].device == p.device:
        return cache[1]
    with torch.no_grad():
        if stem:
            wk = p.detach().contiguous(memory_format=CL)
            out = native.pack_stem_weight(wk, p.shape[2], p.shape[3])
        else:
            src = p.detach()
            if p.dim() == 4:
                src = src.contiguous(memory_format=CL)
                out = torch.empty((p.shape[0], p.shape[1] * p.shape[2] * p.shape[3]), dtype=torch.bfloat16,
                                  device=p.device)
            else:
                src = src.contiguous()
                out = torch.empty(p.shape, dtype=torch.bfloat16, device=p.device)
            native.cast_bf16(src, out)
    p._ddl_cast_cache = (ver, out)
    return out


def _krsc(p: torch.Tensor) -> bool:
    return p.dim() != 4 or p.is_contiguous(memory_format=CL)


# ------------------------------------------------------------------------------------------------
# conv + BN(train/eval) + ReLU (+ residual)
# ------------------------------------------------------------------------------------------------
class _ConvBnAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, gamma, beta, running_mean, running_var, stride, pad, dil, eps, momentum,
                relu, train):
        R, S = weight.shape[2], weight.shape[3]
        wb = weight_bf16(weight)
        # stem: the padded / row-interleaved image the TMA kernels read is built once and shared with the wgrad kernel
        xp = native.stem_prepare(x, (R, S), stride, pad, dil) if (train and x.shape[1] == 4) else None
        y, stats = native.conv_fwd(x, wb, (R, S), stride, pad, dil, stats=train, cout=weight.shape[0], prepadded=xp) \
            if train else (native.conv_fwd(x, wb, (R, S), stride, pad, dil, cout=weight.shape[0]), None)
        use_bits = train and relu and residual is not None
        if use_bits:      # residual layer: 1-bit ReLU mask for backward instead of re-reading z
            z, save, zmask = native.bn_act_fwd(y, stats, gamma, beta, running_mean, running_var, eps, momentum, relu,
                                               residual, train, want_mask=True)
        else:
            z, save = native.bn_act_fwd(y, stats, gamma, beta, running_mean, running_var, eps, momentum, relu, residual,
                                        train)
            zmask = None
        ctx.cfg = (stride, pad, dil, relu, residual is not None, (R, S))
        ctx.params = (weight, gamma, beta)
        if train:
            # wb is a view of the engine's bf16 weight arena: kept as a plain attribute (no autograd
            # version check) — the arena is only rewritten by the bucket kernel, which is ordered after
            # this layer's backward (see notify_ready at the end of backward)
            ctx.wb = wb
            ctx.xp = xp
            ctx.save_for_backward(x, y, zmask if use_bits else z, save)
        return z

    @staticmethod
    def backward(ctx, dz):
        stride, pad, dil, relu, has_res, kernel = ctx.cfg
        weight, gamma, beta = ctx.params
        x, y, z, save = ctx.saved_tensors
        zmask = z if (z is not None and z.dtype == torch.uint8) else None     # residual layers saved the bit mask
        wb = ctx.wb
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)
        gg = grad_buffer(gamma) if gamma.requires_grad else None
        bg = grad_buffer(beta) if beta.requires_grad else None
        dy, dres, _ = native.bn_act_bwd(dz, None if zmask is not None else z, y, save, gamma, relu,
                                        has_res and ctx.needs_input_grad[1], gg, bg, beta=beta, had_residual=has_res,
                                        zmask=zmask)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = native.conv_dgrad(dy, wb, x.shape, kernel, stride, pad, dil)
        if weight.requires_grad:
            gw = grad_buffer(weight)
            xp = ctx.xp
            run_wgrad(weight, lambda: native.conv_wgrad(x, dy, gw, kernel, stride, pad, dil, prepadded=xp), x, dy,
                      *((xp,) if xp is not None else ()))
        # LAST: a ready bucket may launch its allreduce+update kernel on the side stream now; everything
        # this layer still needed from the weight arenas (gamma, wb) has been enqueued before the event
        if gamma.requires_grad:
            notify_ready(gamma)
            notify_ready(beta)
        if weight.requires_grad:
            notify_ready(weight)
        return (dx, dres) + (None,) * 12


def conv_bn_act(x, weight, gamma, beta, running_mean, running_var, stride=1, pad=0, dil=1, eps=1e-5, momentum=0.1,
                relu=True, residual=None, training=True):
    """z = act(BN(conv(x, weight)) [+ residual])  — the unit every ResNet/Inception layer is made of."""
    if use_native(x) and native.supports_conv(x.shape[1], weight.shape[0]) \
            and native.bn_supported(weight.shape[0]) and _krsc(weight):
        return _ConvBnAct.apply(x, residual, weight, gamma, beta, running_mean, running_var, stride, pad, dil, eps,
                                momentum, relu, training)
    xi = x[:, : weight.shape[1]] if x.shape[1] != weight.shape[1] else x     # NHWC4 stem input on the composite path
    y = F.conv2d(xi.to(weight.dtype) if not x.is_cuda else xi, weight.to(xi.dtype) if x.is_cuda else weight, None,
                 stride, pad, dil)
    z = F.batch_norm(y.float(), running_mean, running_var, gamma, beta, training, momentum, eps).to(y.dtype)
    if residual is not None:
        z = z + residual
    return F.relu(z) if relu else z


# ------------------------------------------------------------------------------------------------
# stem: conv + BN(train) + ReLU + max-pool as one unit (ResNet / DenseNet first layers)
# ------------------------------------------------------------------------------------------------
class _ConvBnActPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, stride, pad, dil, eps, momentum, pk, ps, pp):
        R, S = weight.shape[2], weight.shape[3]
        wb = weight_bf16(weight)
        y, stats = native.conv_fwd(x, wb, (R, S), stride, pad, dil, stats=True, cout=weight.shape[0])
        pooled, arg, save = native.bn_relu_maxpool_fwd(y, stats, gamma, beta, running_mean, running_var, eps, momentum,
                                                       pk, ps, pp)
        ctx.cfg = (stride, pad, dil, (R, S), (pk, ps, pp))
        ctx.params = (weight, gamma, beta)
        ctx.wb = wb
        ctx.save_for_backward(x, y, arg, save)
        return pooled

    @staticmethod
    def backward(ctx, dpooled):
        stride, pad, dil, kernel, (pk, ps, pp) = ctx.cfg
        weight, gamma, beta = ctx.params
        x, y, arg, save = ctx.saved_tensors
        if not dpooled.is_contiguous(memory_format=CL):
            dpooled = dpooled.contiguous(memory_format=CL)
        gg = grad_buffer(gamma) if gamma.requires_grad else None
        bg = grad_buffer(beta) if beta.requires_grad else None
        dy = native.bn_pool_bwd(dpooled, arg, y, save, gamma, beta, gg, bg, pk, ps, pp)
        dx = native.conv_dgrad(dy, ctx.wb, x.shape, kernel, stride, pad, dil) if ctx.needs_input_grad[0] else None
        if weight.requires_grad:
            gw = grad_buffer(weight)
            run_wgrad(weight, lambda: native.conv_wgrad(x, dy, gw, kernel, stride, pad, dil), x, dy)
        if gamma.requires_grad:
            notify_ready(gamma)
            notify_ready(beta)
        if weight.requires_grad:
            notify_ready(weight)
        return (dx,) + (None,) * 13


# The fused stem trades ~1.2 GB of HBM traffic for ~5 GB of L2 gathers; it is off unless DDL_FUSE_STEM_POOL=1 (which of
# the two is faster on H100 was not measured).
FUSE_STEM_POOL = os.environ.get("DDL_FUSE_STEM_POOL", "0") != "0"


def conv_bn_act_maxpool(x, weight, gamma, beta, running_mean, running_var, stride=1, pad=0, dil=1, eps=1e-5,
                        momentum=0.1, training=True, pool_kernel=3, pool_stride=2, pool_pad=1):
    """maxpool(relu(BN(conv(x)))) — the stem of ResNet / DenseNet.  In training on the native path the BN output (the
    largest activation of the network) is never materialised; everywhere else this is conv_bn_act + max_pool2d."""
    if FUSE_STEM_POOL and training and use_native(x) and native.supports_conv(x.shape[1], weight.shape[0]) \
            and native.bn_supported(weight.shape[0]) and _krsc(weight) and torch.is_grad_enabled():
        return _ConvBnActPool.apply(x, weight, gamma, beta, running_mean, running_var, stride, pad, dil, eps, momentum,
                                    pool_kernel, pool_stride, pool_pad)
    z = conv_bn_act(x, weight, gamma, beta, running_mean, running_var, stride, pad, dil, eps, momentum, True, None,
                    training)
    return max_pool2d(z, pool_kernel, pool_stride, pool_pad)


# ------------------------------------------------------------------------------------------------
# standalone BN(train/eval) + ReLU on a tensor (pre-activation nets: DenseNet's norm -> relu -> conv)
# ------------------------------------------------------------------------------------------------
class _BnAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, eps, momentum, relu, train):
        z, save = native.bn_act_fwd(x, None, gamma, beta, running_mean, running_var, eps, momentum, relu, None, train)
        ctx.relu = relu
        ctx.params = (gamma, beta)
        if train:
            ctx.save_for_backward(x, z, save)
        return z

    @staticmethod
    def backward(ctx, dz):
        gamma, beta = ctx.params
        x, z, save = ctx.saved_tensors
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)
        gg = grad_buffer(gamma) if gamma.requires_grad else None
        bg = grad_buffer(beta) if beta.requires_grad else None
        dx, _, _ = native.bn_act_bwd(dz, z, x, save, gamma, ctx.relu, False, gg, bg, beta=beta, had_residual=False)
        if gamma.requires_grad:
            notify_ready(gamma)
            notify_ready(beta)
        return (dx if ctx.needs_input_grad[0] else None,) + (None,) * 8


def batch_norm_act(x, gamma, beta, running_mean, running_var, eps=1e-5, momentum=0.1, relu=True, training=True):
    """z = act(BN(x)) with the batch statistics reduced by the native channel_stats kernel."""
    if use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and native.bn_supported(x.shape[1]) \
            and (training or not torch.is_grad_enabled()):
        return _BnAct.apply(x, gamma, beta, running_mean, running_var, eps, momentum, relu, training)
    z = F.batch_norm(x.float(), running_mean, running_var, gamma, beta, training, momentum, eps).to(x.dtype)
    return F.relu(z) if relu else z


# ------------------------------------------------------------------------------------------------
# conv + bias + ReLU (VGG / AlexNet)
# ------------------------------------------------------------------------------------------------
class _ConvBiasAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, stride, pad, dil, relu):
        R, S = weight.shape[2], weight.shape[3]
        wb = weight_bf16(weight)
        z = native.conv_fwd(x, wb, (R, S), stride, pad, dil, bias=bias, relu=relu, cout=weight.shape[0])
        ctx.cfg = (stride, pad, dil, relu, (R, S))
        ctx.params = (weight, bias)
        ctx.wb = wb
        ctx.save_for_backward(x, z)
        return z

    @staticmethod
    def backward(ctx, dz):
        stride, pad, dil, relu, kernel = ctx.cfg
        weight, bias = ctx.params
        x, z = ctx.saved_tensors
        wb = ctx.wb
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)
        db = grad_buffer(bias) if (bias is not None and bias.requires_grad) else None
        dy = native.bias_relu_bwd(dz, z, db, relu) if (relu or db is not None) else dz
        dx = native.conv_dgrad(dy, wb, x.shape, kernel, stride, pad, dil) if ctx.needs_input_grad[0] else None
        if weight.requires_grad:
            native.conv_wgrad(x, dy, grad_buffer(weight), kernel, stride, pad, dil)
        if db is not None:
            notify_ready(bias)
        if weight.requires_grad:
            notify_ready(weight)
        return dx, None, None, None, None, None, None


def conv_bias_act(x, weight, bias=None, stride=1, pad=0, dil=1, relu=True):
    if use_native(x) and native.supports_conv(x.shape[1], weight.shape[0]) and _krsc(weight):
        return _ConvBiasAct.apply(x, weight, bias, stride, pad, dil, relu)
    xi = x[:, : weight.shape[1]] if x.shape[1] != weight.shape[1] else x
    w = weight.to(xi.dtype) if x.is_cuda else weight
    b = bias.to(xi.dtype) if (bias is not None and x.is_cuda) else bias
    y = F.conv2d(xi if x.is_cuda else xi.to(weight.dtype), w, b, stride, pad, dil)
    return F.relu(y) if relu else y


# ------------------------------------------------------------------------------------------------
# linear (+bias, +ReLU)
# ------------------------------------------------------------------------------------------------
class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, relu):
        wb = weight_bf16(weight)
        y = native.linear_fwd(x, wb, bias, relu)
        ctx.relu = relu
        ctx.params = (weight, bias)
        ctx.wb = wb
        ctx.save_for_backward(x, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        weight, bias = ctx.params
        x, y = ctx.saved_tensors
        wb = ctx.wb
        dy = dy.contiguous()
        db = grad_buffer(bias) if (bias is not None and bias.requires_grad) else None
        if ctx.relu or db is not None:
            # dy may be wider than the bias (padded logits): the kernel only reduces the valid columns
            dy = native.bias_relu_bwd(dy, y, db, ctx.relu, c_valid=db.numel() if db is not None else None)
        dx = native.linear_dgrad(dy, wb) if ctx.needs_input_grad[0] else None
        if weight.requires_grad:
            native.linear_wgrad(x, dy, grad_buffer(weight))
        if db is not None:
            notify_ready(bias)
        if weight.requires_grad:
            notify_ready(weight)
        return dx, None, None, None


def linear(x, weight, bias=None, relu=False):
    """y = x W^T + b.  On the native path the result keeps its padded width (multiple of 64);
    use ``out_features`` aware consumers (``softmax_cross_entropy``) or slice."""
    if use_native(x) and x.shape[1] % 8 == 0:
        return _Linear.apply(x.contiguous(), weight, bias, relu)
    y = F.linear(x if not x.is_cuda else x, weight.to(x.dtype) if x.is_cuda else weight,
                 (bias.to(x.dtype) if x.is_cuda else bias) if bias is not None else None)
    return F.relu(y) if relu else y


# ------------------------------------------------------------------------------------------------
# channel concatenation
# ------------------------------------------------------------------------------------------------
class _Concat(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *parts):
        ctx.chans = [int(t.shape[1]) for t in parts]
        return native.concat_channels(parts)

    @staticmethod
    def backward(ctx, dy):
        if not dy.is_contiguous(memory_format=CL):
            dy = dy.contiguous(memory_format=CL)
        return tuple(native.split_channels(dy, ctx.chans))


def concat_channels(parts):
    """torch.cat(parts, 1) for NHWC activations (Inception / DenseNet branches; SURVEY.md K20)."""
    parts = list(parts)
    if use_native(parts[0]) and 1 < len(parts) <= 8 and all(t.shape[1] % 8 == 0 and t.dtype == torch.bfloat16
                                                            and t.is_contiguous(memory_format=CL) for t in parts):
        return _Concat.apply(*parts)
    out = torch.cat(parts, 1)
    return out.contiguous(memory_format=CL) if out.is_cuda and out.dim() == 4 else out


# ------------------------------------------------------------------------------------------------
# pooling
# ------------------------------------------------------------------------------------------------
class _MaxPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, stride, pad, ceil_mode):
        y, arg = native.maxpool_fwd(x, k, stride, pad, ceil_mode)
        ctx.cfg = (k, stride, pad, x.shape)
        ctx.save_for_backward(arg)
        return y

    @staticmethod
    def backward(ctx, dy):
        k, stride, pad, shape = ctx.cfg
        (arg,) = ctx.saved_tensors
        if not dy.is_contiguous(memory_format=CL):
            dy = dy.contiguous(memory_format=CL)
        return native.maxpool_bwd(dy, arg, shape, k, stride, pad), None, None, None, None


def max_pool2d(x, k, stride, pad=0, ceil_mode=False):
    if use_native(x) and x.shape[1] % 8 == 0:
        return _MaxPool.apply(x, k, stride, pad, ceil_mode)
    return F.max_pool2d(x, k, stride, pad, ceil_mode=ceil_mode)


class _AvgPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, stride, pad, cip):
        ctx.cfg = (k, stride, pad, cip, x.shape)
        return native.avgpool_fwd(x, k, stride, pad, cip)

    @staticmethod
    def backward(ctx, dy):
        k, stride, pad, cip, shape = ctx.cfg
        if not dy.is_contiguous(memory_format=CL):
            dy = dy.contiguous(memory_format=CL)
        return native.avgpool_bwd(dy, shape, k, stride, pad, cip), None, None, None, None


def avg_pool2d(x, k, stride, pad=0, count_include_pad=True):
    if use_native(x) and x.shape[1] % 8 == 0:
        return _AvgPool.apply(x, k, stride, pad, count_include_pad)
    return F.avg_pool2d(x, k, stride, pad, count_include_pad=count_include_pad)


class _GlobalAvgPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.shape = x.shape
        return native.global_avgpool_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        return native.global_avgpool_bwd(dy, ctx.shape)


def global_avg_pool(x):
    """[N, C, H, W] -> [N, C]"""
    if use_native(x) and x.shape[1] % 8 == 0:
        return _GlobalAvgPool.apply(x)
    return x.float().mean(dim=(2, 3)).to(x.dtype)


# ------------------------------------------------------------------------------------------------
# dropout (Philox mask recomputed in backward)
# ------------------------------------------------------------------------------------------------
_DROPOUT_STATE = {"seed": 0x5EED, "offset": 0, "step": {}}


def seed_dropout(seed: int) -> None:
    _DROPOUT_STATE["seed"] = int(seed)
    _DROPOUT_STATE["offset"] = 0


def _dropout_step(device) -> torch.Tensor:
    """Device-resident step counter mixed into the Philox key (one per device, created on first use)."""
    key = device.index or 0
    t = _DROPOUT_STATE["step"].get(key)
    if t is None:
        t = _DROPOUT_STATE["step"][key] = torch.zeros((), dtype=torch.int64, device=device)
    return t


def advance_dropout_step() -> None:
    """Advance the device-side dropout step counters (no-op when no dropout layer ran on a GPU yet).  The host-side
    offset already makes eager steps draw fresh masks; a step replayed from a CUDA graph freezes every launch
    argument, so ``GraphedStep`` ends each captured step with this one-element increment instead."""
    for t in _DROPOUT_STATE["step"].values():
        t.add_(1)


class _Dropout(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p):
        seed, off = _DROPOUT_STATE["seed"], _DROPOUT_STATE["offset"]
        _DROPOUT_STATE["offset"] = off + (x.numel() + 7) // 8
        # the Philox mask is indexed by memory offset: keep NHWC activations in their own (dense) memory order and
        # make the gradient follow the same order in backward
        cl = x.dim() == 4 and x.is_contiguous(memory_format=CL)
        step = _dropout_step(x.device)
        ctx.cfg = (p, seed, off, cl, step)
        return native.dropout(x if cl else x.contiguous(), p, seed, off, step)

    @staticmethod
    def backward(ctx, dy):
        p, seed, off, cl, step = ctx.cfg
        dy = dy.contiguous(memory_format=CL) if cl else dy.contiguous()
        return native.dropout(dy, p, seed, off, step), None


def dropout(x, p=0.5, training=True):
    if not training or p <= 0.0:
        return x
    if use_native(x) and x.numel() % 8 == 0:
        return _Dropout.apply(x, p)
    return F.dropout(x, p, training)


# ------------------------------------------------------------------------------------------------
# softmax cross-entropy (+ top-k counters)
# ------------------------------------------------------------------------------------------------
class _SoftmaxXent(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, classes):
        loss, dlog, _ = native.softmax_xent(logits if logits.stride(1) == 1 else logits.contiguous(), labels, classes,
                                            want_grad=True)
        ctx.save_for_backward(dlog)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        (dlog,) = ctx.saved_tensors
        # dloss is 1.0 in every training loop of this repo; honour other values without a sync
        return dlog * dloss.to(dlog.dtype), None, None


def softmax_cross_entropy(logits, labels, classes: Optional[int] = None):
    """Mean cross-entropy.  ``logits`` may be wider than ``classes`` (padded FC output)."""
    classes = classes or logits.shape[1]
    if use_native(logits) and logits.dtype == torch.bfloat16:
        return _SoftmaxXent.apply(logits, labels, classes)
    return F.cross_entropy(logits[:, :classes].float(), labels)


def topk_correct(logits, labels, classes: Optional[int] = None):
    """int32[2] = (#top-1 hits, #top-5 hits) without a host sync."""
    classes = classes or logits.shape[1]
    if use_native(logits) and logits.dtype == torch.bfloat16:
        lg = logits.detach()
        _, _, corr = native.softmax_xent(lg if lg.stride(1) == 1 else lg.contiguous(), labels, classes, want_grad=False,
                                         count_correct=True)
        return corr
    lg = logits[:, :classes].float()
    _, pred = lg.topk(min(5, classes), 1, True, True)
    hit = pred.eq(labels.view(-1, 1))
    return torch.stack([hit[:, :1].sum(), hit.sum()]).to(torch.int32)
