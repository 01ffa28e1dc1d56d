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


def is_stem_weight(p: torch.Tensor, groups: Optional[int] = None) -> bool:
    """A first-layer conv weight on an NHWC4 image (Cin <= 4), which the stem kernels take re-packed.  A grouped weight
    ``[Cout, Cin/groups, R, S]`` can have as few input channels per group (ResNeXt-50's ``[128, 4, 3, 3]``) and is not
    one: ``groups`` defaults to the ``_ddl_groups`` attribute ``models.layers.Conv2d`` puts on its weight."""
    g = groups if groups is not None else getattr(p, "_ddl_groups", 1)
    return p.dim() == 4 and p.shape[1] <= 4 and g == 1


def weight_bf16(p: torch.Tensor, kernel: Optional[Tuple[int, int]] = None, groups: Optional[int] = None,
                stem: Optional[bool] = None) -> torch.Tensor:
    """bf16 GEMM operand of a parameter.

    With a fused engine attached the copy is a view into the bf16 weight arena that the
    allreduce+SGD kernel refreshes every step (no per-step cast).  Otherwise it is cast on
    demand and cached against the parameter's version counter.  Stem weights (Cin <= 4) are
    re-packed to the padded [Cout, KB*64] matrix.  Grouped weights come as the compact
    [Cout, R*S*Cin/groups] matrix (``native.expand_grouped_weight`` derives the kernels' operand from it).
    ``stem=False``: a weight with <= 4 input channels that is not an image convolution (a squeeze-excitation fc2 with a
    squeeze width of 4) keeps the plain [Cout, Cin*R*S] layout.
    """
    stem = is_stem_weight(p, groups) if stem is None else stem
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
                relu, train, groups, sample_scale=None):
        R, S = weight.shape[2], weight.shape[3]
        wb = weight_bf16(weight, groups=groups)
        if groups > 1:      # this step's block-diagonal operand, shared by the forward and the data gradient
            wb = native.expand_grouped_weight(wb, R * S, groups)
        # stem: the padded / row-interleaved image the TMA kernels read is built once and shared with the wgrad kernel
        xp = native.stem_prepare(x, (R, S), stride, pad, dil) if (train and x.shape[1] == 4 and groups == 1) else None
        y, stats = native.conv_fwd(x, wb, (R, S), stride, pad, dil, stats=train, cout=weight.shape[0], prepadded=xp,
                                   groups=groups) \
            if train else (native.conv_fwd(x, wb, (R, S), stride, pad, dil, cout=weight.shape[0], groups=groups), None)
        use_bits = train and relu and relu != 2 and residual is not None
        if use_bits:      # residual layer: 1-bit ReLU mask for backward instead of re-reading z
            z, save, zmask = native.bn_act_fwd(y, stats, gamma, beta, running_mean, running_var, eps, momentum, relu,
                                               residual, train, want_mask=True)
        else:
            z, save = native.bn_act_fwd(y, stats, gamma, beta, running_mean, running_var, eps, momentum, relu, residual,
                                        train, sample_scale=sample_scale)
            zmask = None
        ctx.cfg = (stride, pad, dil, relu, residual is not None, (R, S), groups)
        ctx.sample_scale = sample_scale
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
        stride, pad, dil, relu, has_res, kernel, groups = ctx.cfg
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
                                        zmask=zmask, sample_scale=ctx.sample_scale)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = native.conv_dgrad(dy, wb, x.shape, kernel, stride, pad, dil, groups=groups)
        if weight.requires_grad:
            gw = grad_buffer(weight)
            xp = ctx.xp
            run_wgrad(weight, lambda: native.conv_wgrad(x, dy, gw, kernel, stride, pad, dil, prepadded=xp, groups=groups),
                      x, dy, *((xp,) if xp is not None else ()))
        # LAST: a ready bucket may launch its allreduce+update kernel on the side stream now; everything
        # this layer still needed from the weight arenas (gamma, wb) has been enqueued before the event
        for p in (gamma, beta, weight):
            if p.requires_grad:
                notify_ready(p)
        return (dx, dres) + (None,) * 14


def conv_bn_act(x, weight, gamma, beta, running_mean, running_var, stride=1, pad=0, dil=1, eps=1e-5, momentum=0.1,
                relu=True, residual=None, training=True, groups=1, relu6=False, hardswish=False, silu=False,
                sample_scale=None, gelu=False):
    """z = act(BN(conv(x, weight)) [+ residual])  — the unit every ResNet/Inception layer is made of.  ``groups`` > 1:
    grouped convolution (``weight`` is [Cout, Cin/groups, R, S]); depthwise shapes that ``native.supports_depthwise`` (3x3)
    or ``native.supports_depthwise5`` (5x5) accept run on the depthwise kernels, other shapes outside ``native.supports_grouped`` take the composite path.
    ``relu6``: the activation is ReLU6 (clamp to [0, 6]) instead of ``relu``; ``hardswish``: it is hardswish
    (v * clamp(v + 3, 0, 6) / 6), which takes no ``residual``; ``silu``: it is SiLU (v * sigmoid(v)), which takes no
    ``residual`` either; ``gelu``: it is GELU (v * Phi(v), the erf form), with the same restriction.  ``sample_scale``: fp32 [N] per-sample scales of stochastic depth (``stochastic_depth_keep``):
    z = BN(conv(x)) * sample_scale[n] + residual, with a ``residual``, no activation and in training; the batch
    statistics cover every sample, dropped ones included."""
    if hardswish and (relu6 or residual is not None):
        raise ValueError("conv_bn_act: hardswish is neither combined with relu6 nor with a residual")
    if silu and (relu6 or hardswish or residual is not None):
        raise ValueError("conv_bn_act: SiLU is neither combined with relu6 / hardswish nor with a residual")
    if gelu and (relu6 or hardswish or silu or residual is not None):
        raise ValueError("conv_bn_act: GELU is neither combined with another activation nor with a residual")
    if sample_scale is not None and (residual is None or relu or relu6 or hardswish or silu or gelu or not training):
        raise ValueError("conv_bn_act: sample_scale needs a residual, no activation and training")
    act = 5 if gelu else (4 if silu else (3 if hardswish else (2 if relu6 else relu)))
    if use_native(x) and sample_scale is not None:
        if not (native.supports_conv(x.shape[1], weight.shape[0]) and groups == 1 and native.bn_supported(weight.shape[0])
                and _krsc(weight)):
            raise ValueError("conv_bn_act: stochastic depth is fused for dense convolutions with a multiple of 8 "
                             "output channels only")
        return _ConvBnAct.apply(x, residual, weight, gamma, beta, running_mean, running_var, stride, pad, dil, eps,
                                momentum, act, training, groups, sample_scale)
    if use_native(x) and groups > 1 and x.shape[1] == weight.shape[0] and weight.shape[1] == 1 \
            and native.depthwise_native(weight.shape[0], tuple(weight.shape[2:]), stride, pad, dil, groups) \
            and _krsc(weight):
        return _DwConvBnAct.apply(x, residual, weight, gamma, beta, running_mean, running_var, stride, eps, momentum,
                                  act, training)
    if use_native(x) and native.supports_conv(x.shape[1], weight.shape[0]) \
            and (groups == 1 or native.supports_grouped(x.shape[1], weight.shape[0], groups)) \
            and native.bn_supported(weight.shape[0]) and _krsc(weight):
        return _ConvBnAct.apply(x, residual, weight, gamma, beta, running_mean, running_var, stride, pad, dil, eps,
                                momentum, act, training, groups)
    xi = x[:, : weight.shape[1]] if (x.shape[1] != weight.shape[1] and groups == 1) else x   # NHWC4 stem input
    y = F.conv2d(xi.to(weight.dtype) if not x.is_cuda else xi, weight.to(xi.dtype) if x.is_cuda else weight, None,
                 stride, pad, dil, groups)
    z = F.batch_norm(y.float(), running_mean, running_var, gamma, beta, training, momentum, eps).to(y.dtype)
    if sample_scale is not None:
        z = z * sample_scale.to(z.dtype).view(-1, 1, 1, 1)
    if residual is not None:
        z = z + residual
    if gelu:
        return F.gelu(z)
    if silu:
        return F.silu(z)
    if hardswish:
        return F.hardswish(z)
    if relu6:
        return F.relu6(z)
    return F.relu(z) if relu else z


# ------------------------------------------------------------------------------------------------
# depthwise 3x3 / 5x5 conv + BN(train/eval) + ReLU / ReLU6 / hardswish (+ residual)  (MobileNetV2 / V3)
# ------------------------------------------------------------------------------------------------
class _DwConvBnAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, gamma, beta, running_mean, running_var, stride, eps, momentum, relu, train):
        k = weight.shape[2]
        wb = weight_bf16(weight, groups=weight.shape[0])          # [C, k*k]
        y, stats = native.dwconv_fwd(x, wb, stride, stats=True, k=k) if train else \
            (native.dwconv_fwd(x, wb, stride, k=k), None)
        z, save = native.bn_act_fwd(y, stats, gamma, beta, running_mean, running_var, eps, momentum, relu, residual,
                                    train)
        ctx.cfg = (stride, relu, residual is not None, k)
        ctx.params = (weight, gamma, beta)
        if train:
            ctx.wb = wb       # view of the bf16 weight arena: see _ConvBnAct
            ctx.save_for_backward(x, y, z, save)
        return z

    @staticmethod
    def backward(ctx, dz):
        stride, relu, has_res, k = ctx.cfg
        weight, gamma, beta = ctx.params
        x, y, z, save = ctx.saved_tensors
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)
        gg = grad_buffer(gamma) if gamma.requires_grad else None
        bg = grad_buffer(beta) if beta.requires_grad else None
        dy, dres, _ = native.bn_act_bwd(dz, z, y, save, gamma, relu, has_res and ctx.needs_input_grad[1], gg, bg,
                                        beta=beta, had_residual=has_res)
        dx = native.dwconv_dgrad(dy, ctx.wb, x.shape, stride, k=k) if ctx.needs_input_grad[0] else None
        if weight.requires_grad:
            gw = grad_buffer(weight)
            run_wgrad(weight, lambda: native.dwconv_wgrad(x, dy, gw, stride, k=k), x, dy)
        for p in (gamma, beta, weight):       # LAST, as in _ConvBnAct
            if p.requires_grad:
                notify_ready(p)
        return (dx, dres) + (None,) * 10


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
        for p in (gamma, beta, weight):
            if p.requires_grad:
                notify_ready(p)
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
        for p in (gamma, beta):
            if p.requires_grad:
                notify_ready(p)
        return (dx if ctx.needs_input_grad[0] else None,) + (None,) * 8


def batch_norm_act(x, gamma, beta, running_mean, running_var, eps=1e-5, momentum=0.1, relu=True, training=True,
                   relu6=False):
    """z = act(BN(x)) with the batch statistics reduced by the native channel_stats kernel (``relu6``: ReLU6)."""
    if use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and native.bn_supported(x.shape[1]) \
            and (training or not torch.is_grad_enabled()):
        return _BnAct.apply(x, gamma, beta, running_mean, running_var, eps, momentum, 2 if relu6 else relu, training)
    z = F.batch_norm(x.float(), running_mean, running_var, gamma, beta, training, momentum, eps).to(x.dtype)
    if relu6:
        return F.relu6(z)
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


def conv_bias_act(x, weight, bias=None, stride=1, pad=0, dil=1, relu=True, groups=1):
    """Stand-alone conv (+ bias, + ReLU); grouped convolutions (no BN after them) run on the composite path."""
    if use_native(x) and groups == 1 and native.supports_conv(x.shape[1], weight.shape[0]) and _krsc(weight):
        return _ConvBiasAct.apply(x, weight, bias, stride, pad, dil, relu)
    xi = x[:, : weight.shape[1]] if (x.shape[1] != weight.shape[1] and groups == 1) else x
    w = weight.to(xi.dtype) if x.is_cuda else weight
    b = bias.to(xi.dtype) if (bias is not None and x.is_cuda) else bias
    y = F.conv2d(xi if x.is_cuda else xi.to(weight.dtype), w, b, stride, pad, dil, groups)
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
# hardswish on [B, F] (MobileNetV3's classifier)
# ------------------------------------------------------------------------------------------------
class _Hardswish(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return native.hardswish_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return native.hardswish_bwd(dy.contiguous(), x)


def hardswish(x):
    """x * clamp(x + 3, 0, 6) / 6; the native backward recomputes the gradient from the saved input."""
    if use_native(x) and x.dtype == torch.bfloat16 and x.is_contiguous() and x.numel() % 8 == 0:
        return _Hardswish.apply(x)
    return F.hardswish(x)


# ------------------------------------------------------------------------------------------------
# squeeze-excitation: x * hardsigmoid(fc2(relu(fc1(mean_hw(x)))))  (MobileNetV3)
# ------------------------------------------------------------------------------------------------
class _SqueezeExcite(torch.autograd.Function):
    """One autograd node with a hand-scheduled backward: the gradient of x from the scale path and from the pooling
    path are formed by one kernel (se_apply), not summed by autograd, and the gate gradient is one deterministic
    reduction (se_reduce) written straight into the fc2 GEMM's operand layout."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, train):
        w1b, w2b = weight_bf16(w1), weight_bf16(w2)               # [C', C], [C, C'] (the 1x1 conv weights flattened)
        cs = w1.shape[0]
        pooled = native.global_avgpool_fwd(x)                     # [N, C]
        h = native.linear_fwd(pooled, w1b, b1, relu=True)         # [N, C' rounded up to 64], pad columns 0
        hc = h[:, :cs].contiguous()                               # fc2 takes exactly C' inputs
        s = native.linear_fwd(hc, w2b, b2)                        # [N, C rounded up to 64]: the gate logits
        y = native.se_scale(x, s)
        ctx.params = (w1, b1, w2, b2)
        if train:
            ctx.wb = (w1b, w2b)       # views of the bf16 weight arena: see _ConvBnAct
            ctx.save_for_backward(x, pooled, h, hc, s)
        return y

    @staticmethod
    def backward(ctx, dy):
        w1, b1, w2, b2 = ctx.params
        x, pooled, h, hc, s = ctx.saved_tensors
        w1b, w2b = ctx.wb
        if not dy.is_contiguous(memory_format=CL):
            dy = dy.contiguous(memory_format=CL)
        cs, c = w1.shape[0], w1.shape[1]
        ds = native.se_reduce(dy, x, s)                           # [N, C rounded up to 64], pad columns 0
        db2 = grad_buffer(b2) if b2.requires_grad else None
        if db2 is not None:
            native.bias_relu_bwd(ds, ds, db2, False, c_valid=c)
        dh = native.linear_dgrad(ds, w2b)                         # [N, C']
        if w2.requires_grad:
            native.linear_wgrad(hc, ds, grad_buffer(w2))
        # fc1's output gradient as its GEMM operand: C' rounded up to 64 columns, the pad zero (h is 0 there, so the
        # ReLU mask clears it too)
        dhp = torch.zeros((dh.shape[0], h.shape[1]), dtype=dh.dtype, device=dh.device)
        dhp[:, :cs] = dh
        dhp = native.bias_relu_bwd(dhp, h, grad_buffer(b1) if b1.requires_grad else None, True, c_valid=cs)
        dx = None
        if ctx.needs_input_grad[0]:
            dpooled = native.linear_dgrad(dhp, w1b)               # [N, C]
            dx = native.se_apply(dy, s, dpooled)
        if w1.requires_grad:
            native.linear_wgrad(pooled, dhp, grad_buffer(w1))
        for p in (b2, w2, b1, w1):                                # LAST, as in _ConvBnAct
            if p.requires_grad:
                notify_ready(p)
        return dx, None, None, None, None, None


class _SqueezeExciteSiLU(torch.autograd.Function):
    """x * sigmoid(fc2(silu(fc1(mean_hw(x))))) (EfficientNet) as one node, with _SqueezeExcite's backward schedule.  Any
    squeeze width C': fc2's K = C' is padded with zero columns to C'8 = C' rounded up to 8 (a 16-byte GEMM operand row),
    through a padded bf16 copy of its weight made in forward (so a captured graph rebuilds it from the weight arena every
    replay) and a padded fp32 weight-gradient scratch folded into the compact slot."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, train):
        cs, c = w1.shape[0], w1.shape[1]
        cs8 = _ceil8(cs)
        w1b, w2b = weight_bf16(w1), weight_bf16(w2, stem=False)   # [C', C], [C, C']
        w2p = w2b if cs8 == cs else native.pad_cols_bf16(w2b, cs8)                    # [C, C'8]
        pooled = native.global_avgpool_fwd(x)                     # [N, C]
        h = native.linear_fwd(pooled, w1b, b1)                    # [N, C' rounded up to 64]: fc1 logits, pad columns 0
        a = native.silu_rows_fwd(h, cs8)                          # [N, C'8]: fc2's input, pad columns silu(0) = 0
        s = native.linear_fwd(a, w2p, b2)                         # [N, C rounded up to 64]: the gate logits
        y = native.se_scale(x, s, gate="sigmoid")
        ctx.params = (w1, b1, w2, b2)
        if train:
            ctx.wb = (w1b, w2p)       # views of the bf16 weight arena / this step's padded copy: see _ConvBnAct
            ctx.save_for_backward(x, pooled, h, a, s)
        return y

    @staticmethod
    def backward(ctx, dy):
        w1, b1, w2, b2 = ctx.params
        x, pooled, h, a, s = ctx.saved_tensors
        w1b, w2p = ctx.wb
        if not dy.is_contiguous(memory_format=CL):
            dy = dy.contiguous(memory_format=CL)
        cs, c = w1.shape[0], w1.shape[1]
        cs8 = a.shape[1]
        ds = native.se_reduce(dy, x, s, gate="sigmoid")           # [N, C rounded up to 64], pad columns 0
        if b2.requires_grad:
            native.bias_relu_bwd(ds, ds, grad_buffer(b2), False, c_valid=c)
        da = native.linear_dgrad(ds, w2p)                         # [N, C'8]
        if w2.requires_grad:
            if cs8 == cs:
                native.linear_wgrad(a, ds, grad_buffer(w2))
            else:
                gw = native.zeros_f32((c, cs8), ds.device)
                native.linear_wgrad(a, ds, gw)
                native.fold_cols_f32(gw, grad_buffer(w2))
        dh = native.silu_rows_bwd(da, h, cs)                      # [N, C' rounded up to 64]: fc1's GEMM operand, pad 0
        if b1.requires_grad:
            native.bias_relu_bwd(dh, dh, grad_buffer(b1), False, c_valid=cs)
        dx = None
        if ctx.needs_input_grad[0]:
            dpooled = native.linear_dgrad(dh, w1b)                # [N, C]
            dx = native.se_apply(dy, s, dpooled, gate="sigmoid")
        if w1.requires_grad:
            native.linear_wgrad(pooled, dh, grad_buffer(w1))
        for p in (b2, w2, b1, w1):                                # LAST, as in _ConvBnAct
            if p.requires_grad:
                notify_ready(p)
        return dx, None, None, None, None, None


def _ceil8(n: int) -> int:
    return (n + 7) // 8 * 8


def squeeze_excite(x, w1, b1, w2, b2, gate="hardsigmoid", act="relu"):
    """x * gate(fc2(act(fc1(mean_hw(x))))) with fc1 / fc2 the 1x1 convolutions ``w1`` [C', C, 1, 1] + ``b1``
    and ``w2`` [C, C', 1, 1] + ``b2`` (torchvision's ``SqueezeExcitation``).  ``gate="hardsigmoid", act="relu"``
    (MobileNetV3): native on NHWC bf16 activations with C and C' multiples of 8.  ``gate="sigmoid", act="silu"``
    (EfficientNet): native with C a multiple of 8 and any C'.  The composite is the CPU path."""
    if (gate, act) not in (("hardsigmoid", "relu"), ("sigmoid", "silu")):
        raise ValueError(f"squeeze_excite: (gate, act) must be ('hardsigmoid', 'relu') or ('sigmoid', 'silu'), "
                         f"got {(gate, act)}")
    cs, c = w1.shape[0], w1.shape[1]
    native_act = use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL) \
        and c % 8 == 0 and x.shape[1] == c
    if native_act and gate == "sigmoid":
        train = torch.is_grad_enabled() and any(t.requires_grad for t in (x, w1, b1, w2, b2))
        return _SqueezeExciteSiLU.apply(x, w1, b1, w2, b2, train)
    if native_act and cs % 8 == 0:
        train = torch.is_grad_enabled() and any(t.requires_grad for t in (x, w1, b1, w2, b2))
        return _SqueezeExcite.apply(x, w1, b1, w2, b2, train)
    dt = x.dtype if x.is_cuda else w1.dtype
    xi = x.to(dt)
    sc = xi.float().mean((2, 3), keepdim=True).to(dt) if x.is_cuda else xi.mean((2, 3), keepdim=True)
    sc = F.conv2d(sc, w1.to(dt), b1.to(dt))
    sc = F.silu(sc) if act == "silu" else F.relu(sc)
    sc = F.conv2d(sc, w2.to(dt), b2.to(dt))
    sc = torch.sigmoid(sc) if gate == "sigmoid" else F.hardsigmoid(sc)
    return xi * sc


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


def stochastic_depth_keep(n: int, p: float, device) -> torch.Tensor:
    """fp32 [n] per-sample scales of stochastic depth ("row" mode): 0 with probability p, else 1 / (1 - p).  On CUDA
    they are drawn on the device from the dropout Philox stream (seed, offset and the device step counter), so a step
    replayed from a CUDA graph draws a fresh vector; the data-parallel rank is mixed into the key, so that the ranks
    drop independent samples of the global batch.  On CPU from torch's generator (the composite path)."""
    device = torch.device(device)
    if device.type != "cuda":
        return torch.empty(n).bernoulli_(1.0 - p).div_(1.0 - p)
    from ..parallel import dist

    seed, off = _DROPOUT_STATE["seed"], _DROPOUT_STATE["offset"]
    _DROPOUT_STATE["offset"] = off + n
    seed = (seed + dist.rank() * 0xD1B54A32D192ED03) & 0xFFFFFFFFFFFFFFFF
    return native.stochastic_depth_keep(n, p, seed, off, _dropout_step(device), device)


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
