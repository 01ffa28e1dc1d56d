"""Swin Transformer (V1) ops: shifted-window attention, the whole ``SwinTransformerBlock`` as ONE autograd node, and
patch merging as another.

    block (torchvision's ``SwinTransformerBlock``, dropout 0), on the NHWC rows [N*H*W, C] in image order:
    forward   t1 = LN1(x);  qkv = t1 Wqkv^T + bqkv;  o = wattn(qkv);  a = o Wp^T + bp;  x1 = x + keep1[n] * a
              t2 = LN2(x1);  h = t2 W1^T + b1;  g = gelu(h);  y = g W2^T + b2;  z = x1 + keep2[n] * y
    backward  dy = keep2 * dz (+ db2);  dg = dgrad_fc2(dy);  dh = gelu_bwd(dg, h) (+ db1);  dt2 = dgrad_fc1(dh)
              dx1 = LN2_bwd(dt2) + dz  (one kernel);  da = keep1 * dx1 (+ dbp);  do = dgrad_proj(da)
              dqkv, dtable = wattn_bwd(do) (+ dbqkv);  dt1 = dgrad_qkv(dqkv);  dx = LN1_bwd(dt1) + dx1  (one kernel)
    weight gradients on the side stream; each input gradient is written once.

LN1 and the qkv / proj linears act on one token at a time, so they commute with torchvision's roll and window
partition: the native block runs them on the image-order rows, and the window-attention kernels gather each window's
tokens from qkv with index arithmetic and scatter O back in image order (csrc/ops/window_attention.cu).  There is no
roll, partition, reverse or copy.  Stochastic depth + residual is ``layer_scale_fwd`` with a scale of ones.

The composites of torch ops (pad, roll, partition, mask, reverse: exactly torchvision's maths) are the CPU path, the
path of feature maps that need padding, and the float64 oracle of the tests.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from . import native
from .functional import CL, grad_buffer, notify_ready, use_native, weight_bf16
from .vit import _dgrad, _gb, _lin, _wgrad


def relative_position_index(window: int) -> torch.Tensor:
    """torchvision's ``relative_position_index`` (int64 [window^4]): (iy - jy + w - 1) (2w - 1) + (ix - jx + w - 1)."""
    coords = torch.stack(torch.meshgrid(torch.arange(window), torch.arange(window), indexing="ij")).flatten(1)
    rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += window - 1
    rel[:, :, 1] += window - 1
    rel[:, :, 0] *= 2 * window - 1
    return rel.sum(-1).flatten()


# ------------------------------------------------------------------------------------------------
# composites (torchvision's maths)
# ------------------------------------------------------------------------------------------------
def _attend(qkv: torch.Tensor, table: torch.Tensor, heads: int, window: int, shift) -> torch.Tensor:
    """Shifted-window attention on the padded qkv map [B, pH, pW, 3C]: roll by -shift, partition, attention with the
    relative-position bias and the shifted-window mask, reverse, roll back.  Returns [B, pH, pW, C]."""
    B, pH, pW, c3 = qkv.shape
    C, w = c3 // 3, window
    L, nW = w * w, (pH // w) * (pW // w)
    if sum(shift) > 0:
        qkv = torch.roll(qkv, shifts=(-shift[0], -shift[1]), dims=(1, 2))
    t = qkv.view(B, pH // w, w, pW // w, w, c3).permute(0, 1, 3, 2, 4, 5).reshape(B * nW, L, c3)
    t = t.reshape(B * nW, L, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = t[0], t[1], t[2]
    attn = (q * (C // heads) ** -0.5).matmul(k.transpose(-2, -1))
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


def _pad_hw(x: torch.Tensor, window: int) -> torch.Tensor:
    """Zero-pad [B, H, W, C] on the bottom / right to multiples of the window (torchvision's F.pad)."""
    H, W = x.shape[1], x.shape[2]
    return F.pad(x, (0, 0, 0, (window - W % window) % window, 0, (window - H % window) % window))


# ------------------------------------------------------------------------------------------------
# the attention functional
# ------------------------------------------------------------------------------------------------
class _WindowAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, table, heads, N, H, W, shift):
        o, lse = native.window_attention_fwd(qkv, table, heads, N, H, W, shift)
        ctx.save_for_backward(qkv, table, o, lse)
        ctx.dims = (heads, N, H, W, shift)
        return o

    @staticmethod
    def backward(ctx, do):
        qkv, table, o, lse = ctx.saved_tensors
        heads, N, H, W, shift = ctx.dims
        dtable = torch.zeros_like(table) if ctx.needs_input_grad[1] else None
        dqkv = native.window_attention_bwd(do.contiguous(), qkv, table, o, lse, heads, N, H, W, shift, dtable)
        return dqkv, dtable, None, None, None, None, None


def window_attention_native(qkv: torch.Tensor, heads: int, H: int, W: int, window: int) -> bool:
    """Whether :func:`window_attention` runs on the native kernels for this input."""
    return (use_native(qkv) and qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.shape[1] % 3 == 0
            and (qkv.shape[1] // 3) % heads == 0
            and native.supports_window_attention(H, W, window, heads, qkv.shape[1] // 3 // heads))


def window_attention(qkv: torch.Tensor, table: torch.Tensor, heads: int, H: int, W: int, window: int = 7,
                     shift: int = 0) -> torch.Tensor:
    """torchvision's shifted-window attention from the qkv rows [N*H*W, 3C] of an NHWC map in image order (head h's
    Q, K, V at columns d h, C + d h, 2C + d h) with the relative-position bias ``table`` [(2w-1)^2, heads]: returns the
    attention output rows [N*H*W, C] in image order, the input of ``proj``.  The shift is set to 0 on a side whose
    padded size is at most the window, as torchvision does; a map that needs padding is zero-padded in qkv (torchvision
    pads the block input, so this equals its maths when the qkv linear has no bias).  Native for bf16 CUDA input with
    window 7, head dim 32 and H, W multiples of 7."""
    N = qkv.shape[0] // (H * W)
    if window_attention_native(qkv, heads, H, W, window):
        return _WindowAttention.apply(qkv.contiguous(), table, heads, N, H, W, shift)
    c3 = qkv.shape[1]
    t = _pad_hw(qkv.reshape(N, H, W, c3), window)
    sh = native.window_shift(H, W, window, shift)
    o = _attend(t, table.to(qkv.dtype) if qkv.is_cuda else table, heads, window, sh)
    return o[:, :H, :W, :].reshape(N * H * W, c3 // 3)


# ------------------------------------------------------------------------------------------------
# the Swin block
# ------------------------------------------------------------------------------------------------
_ONES = {}


def _ones(C: int, device) -> torch.Tensor:
    """fp32 [C] ones: the layer scale of the stochastic-depth + residual kernels (created once per width, eagerly)."""
    key = (C, str(device))
    if key not in _ONES:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("swin_block: run one eager step before capturing a CUDA graph")
        _ONES[key] = torch.ones(C, dtype=torch.float32, device=device)
    return _ONES[key]


def _rows4(x: torch.Tensor) -> torch.Tensor:
    """NHWC activation [N, C, H, W] -> its rows [N*H*W, C] (a view)."""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def _act4(rows: torch.Tensor, N: int, H: int, W: int) -> torch.Tensor:
    """Rows [N*H*W, C] -> the NHWC activation [N, C, H, W] (a view)."""
    return rows.view(N, H, W, rows.shape[1]).permute(0, 3, 1, 2)


def _attn_fwd(qkv, table, heads, N, H, W, shift, part):
    if part is None:
        return native.window_attention_fwd(qkv, table, heads, N, H, W, shift)
    return native.grid_attention_fwd(qkv, table, heads, N, H, W, part[1], grid=part[0])


def _attn_bwd(do, qkv, table, o, lse, heads, N, H, W, shift, part, grad_table):
    if part is None:
        return native.window_attention_bwd(do, qkv, table, o, lse, heads, N, H, W, shift, grad_table)
    return native.grid_attention_bwd(do, qkv, table, o, lse, heads, N, H, W, part[1], grad_table, grid=part[0])


class _SwinBlock(torch.autograd.Function):
    """``part`` None: Swin's shifted-window attention (window_attention.cu).  ``part`` (grid, scale): MaxViT's
    partition attention (the same file's kernels), grid or window partition, logits scaled by ``scale``, no shift."""

    @staticmethod
    def forward(ctx, x, keep1, keep2, heads, shift, part, eps, train, n1_w, n1_b, qkv_w, qkv_b, proj_w, proj_b, table,
                n2_w, n2_b, w1, b1, w2, b2):
        N, C, H, W = x.shape
        x2 = _rows4(x)
        wq, wp, w1b, w2b = weight_bf16(qkv_w), weight_bf16(proj_w), weight_bf16(w1), weight_bf16(w2)
        ones = _ones(C, x.device)
        t1, mean1, rstd1 = native.layer_norm_fwd(x2, n1_w, n1_b, eps)
        qkv = _lin(t1, wq, qkv_b, 3 * C, N)
        o, lse = _attn_fwd(qkv, table, heads, N, H, W, shift, part)
        a = _lin(o, wp, proj_b, C, N)
        x1 = native.layer_scale_fwd(_act4(a, N, H, W), ones, keep1, x)
        x1r = _rows4(x1)
        t2, mean2, rstd2 = native.layer_norm_fwd(x1r, n2_w, n2_b, eps)
        h = _lin(t2, w1b, b1, w1.shape[0], N)
        g = native.gelu_fwd(h)
        y = _lin(g, w2b, b2, C, N)
        z = native.layer_scale_fwd(_act4(y, N, H, W), ones, keep2, x1)
        ctx.params = (n1_w, n1_b, qkv_w, qkv_b, proj_w, proj_b, table, n2_w, n2_b, w1, b1, w2, b2)
        ctx.dims = (N, C, H, W, heads, shift, part)
        ctx.keep = (keep1, keep2)
        if train:
            ctx.wb = (wq, wp, w1b, w2b)   # views of the bf16 weight arena: see functional._ConvBnAct
            ctx.save_for_backward(x2, t1, mean1, rstd1, qkv, o, lse, x1r, t2, mean2, rstd2, h, g)
        return z

    @staticmethod
    def backward(ctx, dz):
        n1_w, n1_b, qkv_w, qkv_b, proj_w, proj_b, table, n2_w, n2_b, w1, b1, w2, b2 = ctx.params
        x2, t1, mean1, rstd1, qkv, o, lse, x1r, t2, mean2, rstd2, h, g = ctx.saved_tensors
        wq, wp, w1b, w2b = ctx.wb
        N, C, H, W, heads, shift, part = ctx.dims
        keep1, keep2 = ctx.keep
        ones = _ones(C, dz.device)
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)
        # y is only read for the layer-scale gradient, which is not wanted: dz stands in for it
        dy = _rows4(native.layer_scale_bwd(dz, dz, ones, keep2, None, _gb(b2)))
        dg = _dgrad(dy, w2b, w2.shape[1], N)
        _wgrad(w2, g, dy, N)
        dh = native.gelu_bwd(dg, h, _gb(b1))
        dt2 = _dgrad(dh, w1b, C, N)
        _wgrad(w1, t2, dh, N)
        dx1 = native.layer_norm_bwd_add(dt2, x1r, mean2, rstd2, n2_w, _rows4(dz), _gb(n2_w), _gb(n2_b))
        dx1_4 = _act4(dx1, N, H, W)
        da = _rows4(native.layer_scale_bwd(dx1_4, dx1_4, ones, keep1, None, _gb(proj_b)))
        do = _dgrad(da, wp, C, N)
        _wgrad(proj_w, o, da, N)
        dqkv = _attn_bwd(do, qkv, table, o, lse, heads, N, H, W, shift, part, _gb(table))
        if qkv_b.requires_grad:
            native.bias_relu_bwd(dqkv, dqkv, grad_buffer(qkv_b), False)
        dx = None
        if ctx.needs_input_grad[0] or n1_w.requires_grad or n1_b.requires_grad:
            dt1 = _dgrad(dqkv, wq, C, N)
            dx = _act4(native.layer_norm_bwd_add(dt1, x2, mean1, rstd1, n1_w, dx1, _gb(n1_w), _gb(n1_b)), N, H, W)
        _wgrad(qkv_w, t1, dqkv, N)
        for p in (b2, w2, b1, w1, n2_w, n2_b, proj_b, proj_w, table, qkv_b, qkv_w, n1_w, n1_b):   # LAST
            if p.requires_grad:
                notify_ready(p)
        return (dx if ctx.needs_input_grad[0] else None,) + (None,) * 20


def swin_block_native(x: torch.Tensor, heads: int, window: int, w1: torch.Tensor) -> bool:
    """Whether :func:`swin_block` runs on the native node for this input and these weights."""
    if not (use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)):
        return False
    N, C, H, W = x.shape
    return (C % heads == 0 and native.supports_window_attention(H, W, window, heads, C // heads)
            and native.supports_layer_norm(C) and native.supports_conv(C, 3 * C)
            and native.supports_conv(C, w1.shape[0]) and native.supports_conv(w1.shape[0], C))


def swin_block(x: torch.Tensor, heads: int, window: int, shift: int, eps: float, n1_w, n1_b, qkv_w, qkv_b, proj_w,
               proj_b, table, n2_w, n2_b, w1, b1, w2, b2, keep1: Optional[torch.Tensor] = None,
               keep2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torchvision's ``SwinTransformerBlock`` (V1, dropout 0) on the NHWC activation ``x`` [N, C, H, W]:
    x1 = x + keep1[n] * proj(wattn(qkv(LN1(x)))) with the relative-position bias ``table`` [(2w-1)^2, heads] and the
    shift (0 on a side whose padded size is at most the window); returns x1 + keep2[n] * fc2(gelu(fc1(LN2(x1)))).
    ``keep1`` / ``keep2``: independent fp32 [N] stochastic-depth scales (``stochastic_depth_keep``), or None."""
    params = (n1_w, n1_b, qkv_w, qkv_b, proj_w, proj_b, table, n2_w, n2_b, w1, b1, w2, b2)
    if swin_block_native(x, heads, window, w1):
        train = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        return _SwinBlock.apply(x, keep1, keep2, heads, shift, None, eps, train, *params)
    dt = x.dtype if x.is_cuda else n1_w.dtype
    c = (lambda p: p.to(dt)) if x.is_cuda else (lambda p: p)
    N, C, H, W = x.shape
    xs = x.permute(0, 2, 3, 1)
    t = _pad_hw(F.layer_norm(xs, (C,), c(n1_w), c(n1_b), eps), window)
    sh = native.window_shift(H, W, window, shift)
    o = _attend(F.linear(t, c(qkv_w), c(qkv_b)), c(table), heads, window, sh)
    a = F.linear(o, c(proj_w), c(proj_b))[:, :H, :W, :]
    if keep1 is not None:
        a = a * keep1.to(a.dtype).view(-1, 1, 1, 1)
    x1 = xs + a
    y = F.linear(F.gelu(F.linear(F.layer_norm(x1, (C,), c(n2_w), c(n2_b), eps), c(w1), c(b1))), c(w2), c(b2))
    if keep2 is not None:
        y = y * keep2.to(y.dtype).view(-1, 1, 1, 1)
    z = (x1 + y).permute(0, 3, 1, 2)
    return z.contiguous(memory_format=CL) if x.is_cuda else z


# ------------------------------------------------------------------------------------------------
# patch merging
# ------------------------------------------------------------------------------------------------
class _PatchMerging(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, norm_w, norm_b, eps, red_w, train):
        N, C, H, W = x.shape
        wr = weight_bf16(red_w)
        y, mean, rstd = native.patch_merge_fwd(x, norm_w, norm_b, eps)
        out = _lin(y, wr, None, 2 * C, N)
        ctx.params = (norm_w, norm_b, red_w)
        ctx.dims = (N, C, H // 2, W // 2)
        if train:
            ctx.wb = wr
            ctx.save_for_backward(x, y, mean, rstd)
        return _act4(out, N, H // 2, W // 2)

    @staticmethod
    def backward(ctx, dout):
        norm_w, norm_b, red_w = ctx.params
        x, y, mean, rstd = ctx.saved_tensors
        N, C, Ho, Wo = ctx.dims
        if not dout.is_contiguous(memory_format=CL):
            dout = dout.contiguous(memory_format=CL)
        d = _rows4(dout)
        dx = None
        if ctx.needs_input_grad[0] or norm_w.requires_grad or norm_b.requires_grad:
            dy = _dgrad(d, ctx.wb, 4 * C, N)
            dx = native.patch_merge_bwd(dy, x, mean, rstd, norm_w, _gb(norm_w), _gb(norm_b))
        _wgrad(red_w, y, d, N)
        for p in (red_w, norm_w, norm_b):
            if p.requires_grad:
                notify_ready(p)
        return (dx if ctx.needs_input_grad[0] else None,) + (None,) * 5


def patch_merging_native(x: torch.Tensor) -> bool:
    """Whether :func:`patch_merging` runs on the native node for this input."""
    return (use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)
            and native.supports_patch_merge(x.shape[2], x.shape[3], x.shape[1])
            and native.supports_conv(4 * x.shape[1], 2 * x.shape[1]))


def patch_merging(x: torch.Tensor, norm_w: torch.Tensor, norm_b: torch.Tensor, eps: float,
                  red_w: torch.Tensor) -> torch.Tensor:
    """torchvision's ``PatchMerging`` on the NHWC activation ``x`` [N, C, H, W]: the 2x2 gather (x0, x1, x2, x3),
    LayerNorm over 4C (``norm_w`` / ``norm_b`` / ``eps``), then the bias-free reduction ``red_w`` [2C, 4C].  Returns
    [N, 2C, ceil(H/2), ceil(W/2)].  Native for even H and W."""
    if patch_merging_native(x):
        train = torch.is_grad_enabled() and any(t.requires_grad for t in (x, norm_w, norm_b, red_w))
        return _PatchMerging.apply(x, norm_w, norm_b, eps, red_w, train)
    dt = x.dtype if x.is_cuda else norm_w.dtype
    c = (lambda p: p.to(dt)) if x.is_cuda else (lambda p: p)
    t = x.permute(0, 2, 3, 1)
    H, W = t.shape[1], t.shape[2]
    t = F.pad(t, (0, 0, 0, W % 2, 0, H % 2))
    t = torch.cat([t[:, 0::2, 0::2], t[:, 1::2, 0::2], t[:, 0::2, 1::2], t[:, 1::2, 1::2]], -1)
    t = F.linear(F.layer_norm(t, (t.shape[-1],), c(norm_w), c(norm_b), eps), c(red_w))
    z = t.permute(0, 3, 1, 2)
    return z.contiguous(memory_format=CL) if x.is_cuda else z
