"""Swin Transformer V2 ops: scaled-cosine shifted-window attention, the whole ``SwinTransformerBlockV2`` as ONE autograd
node, and ``PatchMergingV2`` as another.

    block (torchvision's ``SwinTransformerBlockV2``, dropout 0, post-norm), on the NHWC rows [N*H*W, C] in image order:
    forward   T = 16 sigmoid(cpb(coords));  qkv = x Wqkv^T + [b_q, 0, b_v];  o = cwattn(qkv, T, logit_scale)
              a = o Wp^T + bp;  x1 = x + keep1[n] * LN1(a);  h = x1 W1^T + b1;  y = gelu(h) W2^T + b2
              z = x1 + keep2[n] * LN2(y)
    backward  du2 = keep2 * dz;  dy = LN2_bwd(du2) (+ db2);  dg = dgrad_fc2(dy);  dh = gelu_bwd(dg, h) (+ db1)
              dx1 = dgrad_fc1(dh) + dz  (one kernel);  du1 = keep1 * dx1;  da = LN1_bwd(du1) (+ dbp);  do = dgrad_proj(da)
              dqkv, dT, dlogit_scale, db_q, db_v = cwattn_bwd(do);  dcpb = cpb_bwd(dT)
              dx = dgrad_qkv(dqkv) + dx1  (one kernel)
    weight gradients on the side stream; each input gradient is written once.

The qkv and proj linears act on one token at a time, so they commute with torchvision's pad, roll, window partition and
crop: the native block runs them on the image-order rows of the real tokens, and the attention kernels
(csrc/ops/window_attention_v2.cu) gather each window of the padded frame from qkv with index arithmetic.  A padding
token of torchvision's padded block input has q = b_q, k = 0 and v = b_v (the k-bias is zeroed in every forward); the
kernels synthesise those tokens, never store them, and fold the padding tokens' dv into the v-bias gradient.  The k-bias
gradient stays exactly 0.  The CPB MLP (csrc/ops/swin_v2.cu) runs once per block and step inside the node.

The composites of torch ops (pad, roll, partition, normalize, clamp, cpb, mask, reverse, crop: exactly torchvision's
maths) are the CPU path and the float64 oracle of the tests.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from . import native
from .functional import CL, grad_buffer, notify_ready, use_native, weight_bf16
from .swin import _act4, _ones, _pad_hw, _rows4
from .vit import _dgrad, _gb, _lin, _nhwc, _wgrad

_WINDOW = 8


def relative_coords_table(window: int) -> torch.Tensor:
    """torchvision's ``relative_coords_table`` (fp32 [1, 2w-1, 2w-1, 2]): sign(t) log2(|t| + 1) / 3 of the relative
    offsets scaled to [-8, 8]."""
    r = torch.arange(-(window - 1), window, dtype=torch.float32)
    t = torch.stack(torch.meshgrid([r, r], indexing="ij")).permute(1, 2, 0).contiguous().unsqueeze(0)
    t = t / (window - 1) * 8
    return torch.sign(t) * torch.log2(torch.abs(t) + 1.0) / 3.0


def cpb_table(coords: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, heads: int) -> torch.Tensor:
    """16 sigmoid(cpb_mlp(coords)) as [(2w-1)^2, heads] (torch ops: the composite)."""
    return 16 * torch.sigmoid(F.linear(F.relu(F.linear(coords, w1, b1)), w2).view(-1, heads))


# ------------------------------------------------------------------------------------------------
# composites (torchvision's maths)
# ------------------------------------------------------------------------------------------------
def _attend_v2(qkv: torch.Tensor, table: torch.Tensor, logit_scale: torch.Tensor, heads: int, window: int,
               shift) -> torch.Tensor:
    """Cosine shifted-window attention on the padded qkv map [B, pH, pW, 3C]: roll by -shift, partition, cosine logits
    times exp(min(logit_scale, ln 100)) plus the position bias ``table`` [(2w-1)^2, heads] and the shifted-window mask,
    reverse, roll back.  Returns [B, pH, pW, C]."""
    from .swin import relative_position_index

    B, pH, pW, c3 = qkv.shape
    C, w = c3 // 3, window
    L, nW = w * w, (pH // w) * (pW // w)
    if sum(shift) > 0:
        qkv = torch.roll(qkv, shifts=(-shift[0], -shift[1]), dims=(1, 2))
    t = qkv.reshape(B, pH // w, w, pW // w, w, c3).permute(0, 1, 3, 2, 4, 5).reshape(B * nW, L, c3)
    t = t.reshape(B * nW, L, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = t[0], t[1], t[2]
    attn = F.normalize(q, dim=-1) @ F.normalize(k, dim=-1).transpose(-2, -1)
    attn = attn * torch.clamp(logit_scale.view(heads, 1, 1), max=math.log(100.0)).exp()
    idx = relative_position_index(w).to(table.device)
    attn = attn + table[idx].view(L, L, -1).permute(2, 0, 1).contiguous().unsqueeze(0).to(attn.dtype)
    if sum(shift) > 0:
        mask = qkv.new_zeros((pH, pW))
        hs = ((0, -w), (-w, -shift[0]), (-shift[0], None))
        ws = ((0, -w), (-w, -shift[1]), (-shift[1], None))
        count = 0
        for h in hs:
            for s in ws:
                mask[h[0]:h[1], s[0]:s[1]] = count
                count += 1
        mask = mask.view(pH // w, w, pW // w, w).permute(0, 2, 1, 3).reshape(nW, L)
        mask = mask.unsqueeze(1) - mask.unsqueeze(2)
        mask = mask.masked_fill(mask != 0, float(-100.0)).masked_fill(mask == 0, float(0.0))
        attn = attn.view(B, nW, heads, L, L) + mask.unsqueeze(1).unsqueeze(0)
        attn = attn.view(-1, heads, L, L)
    attn = F.softmax(attn, dim=-1)
    o = attn.matmul(v).transpose(1, 2).reshape(B * nW, L, C)
    o = o.view(B, pH // w, pW // w, w, w, C).permute(0, 1, 3, 2, 4, 5).reshape(B, pH, pW, C)
    if sum(shift) > 0:
        o = torch.roll(o, shifts=(shift[0], shift[1]), dims=(1, 2))
    return o


def _k_zeroed(qkv_b: torch.Tensor) -> torch.Tensor:
    """torchvision's clone of qkv.bias with the k slice zeroed (the gradient of that slice is 0)."""
    b = qkv_b.clone()
    C = b.numel() // 3
    b[C:2 * C] = 0
    return b


# ------------------------------------------------------------------------------------------------
# the attention functional
# ------------------------------------------------------------------------------------------------
class _WindowAttentionV2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, table, logit_scale, q_bias, v_bias, heads, N, H, W, shift):
        o, lse = native.window_attention_v2_fwd(qkv, table, logit_scale, q_bias, v_bias, heads, N, H, W, shift)
        ctx.save_for_backward(qkv, table, logit_scale, q_bias, v_bias, o, lse)
        ctx.dims = (heads, N, H, W, shift)
        return o

    @staticmethod
    def backward(ctx, do):
        qkv, table, ls, qb, vb, o, lse = ctx.saved_tensors
        heads, N, H, W, shift = ctx.dims
        C = qkv.shape[1] // 3
        dtable = torch.empty_like(table) if ctx.needs_input_grad[1] else None
        dls = torch.zeros(heads, dtype=torch.float32, device=qkv.device) if ctx.needs_input_grad[2] else None
        db = (torch.zeros(3 * C, dtype=torch.float32, device=qkv.device)
              if ctx.needs_input_grad[3] or ctx.needs_input_grad[4] else None)
        # qkv's rows are given: q_bias / v_bias only fill the padding tokens, so their gradient is the padding tokens'
        dqkv = native.window_attention_v2_bwd(do.contiguous(), qkv, table, ls.contiguous(), qb, vb, o, lse, heads, N, H,
                                              W, shift, dtable, dls, db, bias_pad_only=True)
        return (dqkv, dtable, None if dls is None else dls.view_as(ls), None if db is None else db[:C],
                None if db is None else db[2 * C:], None, None, None, None, None)


def window_attention_v2_native(qkv: torch.Tensor, heads: int, H: int, W: int, window: int) -> bool:
    """Whether :func:`window_attention_v2` runs on the native kernels for this input."""
    return (use_native(qkv) and qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.shape[1] % 3 == 0
            and (qkv.shape[1] // 3) % heads == 0
            and native.supports_window_attention_v2(H, W, window, heads, qkv.shape[1] // 3 // heads))


def window_attention_v2(qkv: torch.Tensor, table: torch.Tensor, logit_scale: torch.Tensor, q_bias: torch.Tensor,
                        v_bias: torch.Tensor, heads: int, H: int, W: int, window: int = 8,
                        shift: int = 0) -> torch.Tensor:
    """torchvision's scaled-cosine shifted-window attention (Swin V2) from the qkv rows [N*H*W, 3C] of an NHWC map in
    image order (head h's Q, K, V at columns d h, C + d h, 2C + d h), the position bias ``table`` [(2w-1)^2, heads]
    (16 sigmoid of the CPB MLP), ``logit_scale`` [heads, 1, 1] and the q / v biases [C] that torchvision's padding
    tokens carry (their k is 0).  Returns the attention output rows [N*H*W, C] in image order, the input of ``proj``.
    The shift is set to 0 on a side whose padded size is at most the window.  Native for bf16 CUDA input with window
    8 and head dim 32, padded maps included."""
    N = qkv.shape[0] // (H * W)
    if window_attention_v2_native(qkv, heads, H, W, window):
        return _WindowAttentionV2.apply(qkv.contiguous(), table.contiguous(), logit_scale, q_bias, v_bias, heads, N, H,
                                        W, shift)
    c3 = qkv.shape[1]
    C = c3 // 3
    t = qkv.reshape(N, H, W, c3)
    pH, pW = -(-H // window) * window, -(-W // window) * window
    if (pH, pW) != (H, W):
        pad = torch.cat([q_bias, torch.zeros_like(q_bias), v_bias]).to(qkv.dtype)
        full = pad.expand(N, pH, pW, c3).clone()
        full[:, :H, :W] = t
        t = full
    sh = native.window_shift(H, W, window, shift)
    dt = qkv.dtype
    o = _attend_v2(t, table.to(dt), logit_scale.to(dt), heads, window, sh)
    return o[:, :H, :W, :].reshape(N * H * W, C)


# ------------------------------------------------------------------------------------------------
# the Swin V2 block
# ------------------------------------------------------------------------------------------------
class _SwinV2Block(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, keep1, keep2, heads, shift, eps, train, coords, logit_scale, qkv_w, qkv_b, proj_w, proj_b,
                c1_w, c1_b, c2_w, n1_w, n1_b, w1, b1, w2, b2, n2_w, n2_b):
        N, C, H, W = x.shape
        x2 = _rows4(x)
        wq, wp, w1b, w2b = weight_bf16(qkv_w), weight_bf16(proj_w), weight_bf16(w1), weight_bf16(w2)
        ones = _ones(C, x.device)
        table, beff = native.cpb_fwd(coords, c1_w, c1_b, c2_w, heads, qkv_b)
        qkv = _lin(x2, wq, beff, 3 * C, N)
        qb, vb = qkv_b[:C], qkv_b[2 * C:]
        o, lse = native.window_attention_v2_fwd(qkv, table, logit_scale, qb, vb, heads, N, H, W, shift)
        a = _lin(o, wp, proj_b, C, N)
        u1, mean1, rstd1 = native.layer_norm_fwd(a, n1_w, n1_b, eps)
        x1 = native.layer_scale_fwd(_act4(u1, N, H, W), ones, keep1, x)
        x1r = _rows4(x1)
        h = _lin(x1r, w1b, b1, w1.shape[0], N)
        g = native.gelu_fwd(h)
        y = _lin(g, w2b, b2, C, N)
        u2, mean2, rstd2 = native.layer_norm_fwd(y, n2_w, n2_b, eps)
        z = native.layer_scale_fwd(_act4(u2, N, H, W), ones, keep2, x1)
        ctx.params = (coords, logit_scale, qkv_w, qkv_b, proj_w, proj_b, c1_w, c1_b, c2_w, n1_w, n1_b, w1, b1, w2, b2,
                      n2_w, n2_b)
        ctx.dims = (N, C, H, W, heads, shift)
        ctx.keep = (keep1, keep2)
        if train:
            ctx.wb = (wq, wp, w1b, w2b)   # views of the bf16 weight arena: see functional._ConvBnAct
            ctx.save_for_backward(x2, qkv, table, o, lse, a, mean1, rstd1, x1r, h, g, y, mean2, rstd2)
        return z

    @staticmethod
    def backward(ctx, dz):
        (coords, ls, qkv_w, qkv_b, proj_w, proj_b, c1_w, c1_b, c2_w, n1_w, n1_b, w1, b1, w2, b2, n2_w,
         n2_b) = ctx.params
        x2, qkv, table, o, lse, a, mean1, rstd1, x1r, h, g, y, mean2, rstd2 = ctx.saved_tensors
        wq, wp, w1b, w2b = ctx.wb
        N, C, H, W, heads, shift = ctx.dims
        keep1, keep2 = ctx.keep
        ones = _ones(C, dz.device)
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)
        du2 = _rows4(native.layer_scale_bwd(dz, dz, ones, keep2, None, None))
        dy = native.layer_norm_bwd(du2, y, mean2, rstd2, n2_w, _gb(n2_w), _gb(n2_b))
        if b2.requires_grad:
            native.bias_relu_bwd(dy, dy, grad_buffer(b2), False)
        dg = _dgrad(dy, w2b, w2.shape[1], N)
        _wgrad(w2, g, dy, N)
        dh = native.gelu_bwd(dg, h, _gb(b1))
        M = dh.shape[0]
        dx1 = _rows4(native.conv_dgrad(_nhwc(dh, N), w1b, (N, C, M // N, 1), (1, 1), 1, 0, add=_nhwc(_rows4(dz), N)))
        _wgrad(w1, x1r, dh, N)
        dx1_4 = _act4(dx1, N, H, W)
        du1 = _rows4(native.layer_scale_bwd(dx1_4, dx1_4, ones, keep1, None, None))
        da = native.layer_norm_bwd(du1, a, mean1, rstd1, n1_w, _gb(n1_w), _gb(n1_b))
        if proj_b.requires_grad:
            native.bias_relu_bwd(da, da, grad_buffer(proj_b), False)
        do = _dgrad(da, wp, C, N)
        _wgrad(proj_w, o, da, N)
        cpb_grads = (_gb(c1_w), _gb(c1_b), _gb(c2_w))
        dtable = torch.empty_like(table) if any(t is not None for t in cpb_grads) else None
        dqkv = native.window_attention_v2_bwd(do, qkv, table, ls, qkv_b[:C], qkv_b[2 * C:], o, lse, heads, N, H, W,
                                              shift, dtable, _gb(ls), _gb(qkv_b))
        if dtable is not None:
            native.cpb_bwd(coords, c1_w, c1_b, c2_w, table, dtable, heads, *cpb_grads)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = _act4(_rows4(native.conv_dgrad(_nhwc(dqkv, N), wq, (N, C, M // N, 1), (1, 1), 1, 0,
                                                add=_nhwc(dx1, N))), N, H, W)
        _wgrad(qkv_w, x2, dqkv, N)
        for p in (n2_b, n2_w, b2, w2, b1, w1, n1_b, n1_w, proj_b, proj_w, c2_w, c1_b, c1_w, ls, qkv_b, qkv_w):   # LAST
            if p.requires_grad:
                notify_ready(p)
        return (dx,) + (None,) * 23


def swin_v2_block_native(x: torch.Tensor, heads: int, window: int, w1: torch.Tensor) -> bool:
    """Whether :func:`swin_v2_block` runs on the native node for this input and these weights."""
    if not (use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)):
        return False
    N, C, H, W = x.shape
    return (C % heads == 0 and native.supports_window_attention_v2(H, W, window, heads, C // heads)
            and native.supports_layer_norm(C) and native.supports_conv(C, 3 * C)
            and native.supports_conv(C, w1.shape[0]) and native.supports_conv(w1.shape[0], C))


def swin_v2_block(x: torch.Tensor, heads: int, window: int, shift: int, eps: float, coords, logit_scale, qkv_w, qkv_b,
                  proj_w, proj_b, c1_w, c1_b, c2_w, n1_w, n1_b, w1, b1, w2, b2, n2_w, n2_b,
                  keep1: Optional[torch.Tensor] = None, keep2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torchvision's ``SwinTransformerBlockV2`` (dropout 0) on the NHWC activation ``x`` [N, C, H, W]:
    x1 = x + keep1[n] * LN1(proj(cwattn(qkv(x)))) with the cosine attention of ``logit_scale`` [heads, 1, 1], the CPB
    MLP (``c1_w`` [512, 2], ``c1_b``, ``c2_w`` [heads, 512]) on ``coords`` (the relative_coords_table buffer) and the
    shift (0 on a side whose padded size is at most the window); returns x1 + keep2[n] * LN2(fc2(gelu(fc1(x1)))).
    The k slice of ``qkv_b`` is ignored, as torchvision zeroes it.  ``keep1`` / ``keep2``: independent fp32 [N]
    stochastic-depth scales (``stochastic_depth_keep``), or None."""
    params = (coords, logit_scale, qkv_w, qkv_b, proj_w, proj_b, c1_w, c1_b, c2_w, n1_w, n1_b, w1, b1, w2, b2, n2_w,
              n2_b)
    if swin_v2_block_native(x, heads, window, w1):
        train = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        return _SwinV2Block.apply(x, keep1, keep2, heads, shift, eps, train, *params)
    dt = x.dtype if x.is_cuda else n1_w.dtype
    c = (lambda p: p.to(dt)) if x.is_cuda else (lambda p: p)
    N, C, H, W = x.shape
    xs = x.permute(0, 2, 3, 1)
    table = cpb_table(coords, c1_w, c1_b, c2_w, heads)
    sh = native.window_shift(H, W, window, shift)
    qkv = F.linear(_pad_hw(xs, window), c(qkv_w), c(_k_zeroed(qkv_b)))
    o = _attend_v2(qkv, c(table), c(logit_scale), heads, window, sh)
    a = F.linear(o, c(proj_w), c(proj_b))[:, :H, :W, :]
    a = F.layer_norm(a, (C,), c(n1_w), c(n1_b), eps)
    if keep1 is not None:
        a = a * keep1.to(a.dtype).view(-1, 1, 1, 1)
    x1 = xs + a
    y = F.linear(F.gelu(F.linear(x1, c(w1), c(b1))), c(w2), c(b2))
    y = F.layer_norm(y, (C,), c(n2_w), c(n2_b), eps)
    if keep2 is not None:
        y = y * keep2.to(y.dtype).view(-1, 1, 1, 1)
    z = (x1 + y).permute(0, 3, 1, 2)
    return z.contiguous(memory_format=CL) if x.is_cuda else z


# ------------------------------------------------------------------------------------------------
# patch merging V2
# ------------------------------------------------------------------------------------------------
class _PatchMergingV2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, red_w, norm_w, norm_b, eps, train):
        N, C, H, W = x.shape
        wr = weight_bf16(red_w)
        gx = native.merge_gather(x)
        r = _lin(gx, wr, None, 2 * C, N)
        out, mean, rstd = native.layer_norm_fwd(r, norm_w, norm_b, eps)
        ctx.params = (red_w, norm_w, norm_b)
        ctx.dims = (N, C, H, W)
        if train:
            ctx.wb = wr
            ctx.save_for_backward(gx, r, mean, rstd)
        return _act4(out, N, H // 2, W // 2)

    @staticmethod
    def backward(ctx, dout):
        red_w, norm_w, norm_b = ctx.params
        gx, r, mean, rstd = ctx.saved_tensors
        N, C, H, W = ctx.dims
        if not dout.is_contiguous(memory_format=CL):
            dout = dout.contiguous(memory_format=CL)
        dr = native.layer_norm_bwd(_rows4(dout), r, mean, rstd, norm_w, _gb(norm_w), _gb(norm_b))
        dx = None
        if ctx.needs_input_grad[0]:
            dx = native.merge_scatter(_dgrad(dr, ctx.wb, 4 * C, N), N, C, H, W)
        _wgrad(red_w, gx, dr, N)
        for p in (norm_b, norm_w, red_w):
            if p.requires_grad:
                notify_ready(p)
        return (dx,) + (None,) * 5


def patch_merging_v2_native(x: torch.Tensor) -> bool:
    """Whether :func:`patch_merging_v2` runs on the native node for this input."""
    if not (use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)):
        return False
    N, C, H, W = x.shape
    return (H % 2 == 0 and W % 2 == 0 and C % 8 == 0 and native.supports_conv(4 * C, 2 * C)
            and native.supports_layer_norm(2 * C))


def patch_merging_v2(x: torch.Tensor, red_w: torch.Tensor, norm_w: torch.Tensor, norm_b: torch.Tensor,
                     eps: float) -> torch.Tensor:
    """torchvision's ``PatchMergingV2`` on the NHWC activation ``x`` [N, C, H, W]: the 2x2 gather (x0, x1, x2, x3), the
    bias-free reduction ``red_w`` [2C, 4C], then LayerNorm over 2C.  Returns [N, 2C, ceil(H/2), ceil(W/2)].  Native
    for even H and W."""
    if patch_merging_v2_native(x):
        train = torch.is_grad_enabled() and any(t.requires_grad for t in (x, red_w, norm_w, norm_b))
        return _PatchMergingV2.apply(x, red_w, norm_w, norm_b, eps, train)
    dt = x.dtype if x.is_cuda else norm_w.dtype
    c = (lambda p: p.to(dt)) if x.is_cuda else (lambda p: p)
    t = x.permute(0, 2, 3, 1)
    H, W = t.shape[1], t.shape[2]
    t = F.pad(t, (0, 0, 0, W % 2, 0, H % 2))
    t = torch.cat([t[:, 0::2, 0::2], t[:, 1::2, 0::2], t[:, 0::2, 1::2], t[:, 1::2, 1::2]], -1)
    t = F.layer_norm(F.linear(t, c(red_w)), (2 * x.shape[1],), c(norm_w), c(norm_b), eps)
    z = t.permute(0, 3, 1, 2)
    return z.contiguous(memory_format=CL) if x.is_cuda else z
