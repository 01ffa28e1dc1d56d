"""Vision Transformer ops: multi-head self-attention, the whole encoder block as ONE autograd node, and the patch / token
embedding as another.

    encoder block (torchvision's ``EncoderBlock``, dropout 0), on the token rows [N*L, C]:
    forward   t1 = LN1(x);  qkv = t1 Win^T + bin;  o = attn(qkv);  a = o Wout^T + bout
              x1, t2 = x + a, LN2(x + a)        (one kernel);  h = t2 W1^T + b1;  g = gelu(h);  y = g W2^T + b2;  z = x1 + y
    backward  dg = dgrad_fc2(dz)  (+ db2 column sum, wgrad fc2 on the side stream);  dh = gelu_bwd(dg, h) (+ db1)
              dt2 = dgrad_fc1(dh);  dx1 = LN2_bwd(dt2) + dz  (one kernel);  do = dgrad_out(dx1) (+ dbout)
              dqkv = attn_bwd(do);  (+ dbin);  dt1 = dgrad_in(dqkv);  dx = LN1_bwd(dt1) + dx1  (one kernel)

The linears are 1x1 conv-GEMMs on the existing kernels (their [out, in] weights are the GEMM operand as they are), the
token rows viewed as an NHWC activation [N, C, L, 1].  The attention kernels read Q, K and V straight out of qkv and write
O in out_proj's input layout (csrc/ops/attention.cu).  The composites of torch ops are the CPU path and the float64
oracle of the tests; their maths is exactly torchvision's.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from . import native
from .functional import grad_buffer, notify_ready, run_wgrad, use_native, weight_bf16


def _nhwc(t: torch.Tensor, n: int) -> torch.Tensor:
    """Rows [N*L, C] as the channels_last activation [N, C, L, 1] the conv-GEMM kernels take (a view)."""
    return t.view(n, t.shape[0] // n, 1, t.shape[1]).permute(0, 3, 1, 2)


def _rows(t: torch.Tensor) -> torch.Tensor:
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _lin(x, wb, bias, cout, n):
    return _rows(native.conv_fwd(_nhwc(x, n), wb, (1, 1), 1, 0, bias=bias, cout=cout))


def _dgrad(dy, wb, cin, n):
    m = dy.shape[0]
    return _rows(native.conv_dgrad(_nhwc(dy, n), wb, (n, cin, m // n, 1), (1, 1), 1, 0))


def _wgrad(w, x, dy, n):
    if w.requires_grad:
        gw = grad_buffer(w)
        run_wgrad(w, lambda: native.conv_wgrad(_nhwc(x, n), _nhwc(dy, n), gw, (1, 1), 1, 0), x, dy)


def _gb(p):
    return grad_buffer(p) if p is not None and p.requires_grad else None


# ------------------------------------------------------------------------------------------------
# multi-head self-attention on the packed in-projection output
# ------------------------------------------------------------------------------------------------
def _attention_composite(qkv: torch.Tensor, num_heads: int) -> torch.Tensor:
    n, L, c3 = qkv.shape
    C = c3 // 3
    d = C // num_heads
    q, k, v = (t.reshape(n, L, num_heads, d).transpose(1, 2) for t in qkv.split(C, dim=2))
    s = torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(d)
    p = torch.softmax(s.to(torch.promote_types(s.dtype, torch.float32)), dim=-1).to(s.dtype)
    return torch.matmul(p, v).transpose(1, 2).reshape(n, L, C)


class _SelfAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, num_heads):
        n, L, c3 = qkv.shape
        flat = qkv.reshape(n * L, c3)
        o, lse = native.attention_fwd(flat, num_heads, L)
        ctx.save_for_backward(flat, o, lse)
        ctx.dims = (n, L, num_heads)
        return o.view(n, L, c3 // 3)

    @staticmethod
    def backward(ctx, do):
        flat, o, lse = ctx.saved_tensors
        n, L, h = ctx.dims
        dqkv = native.attention_bwd(do.contiguous().view(n * L, -1), flat, o, lse, h, L)
        return dqkv.view(n, L, -1), None


def self_attention_native(qkv: torch.Tensor, num_heads: int) -> bool:
    """Whether :func:`self_attention` runs on the native kernels for this input."""
    return (use_native(qkv) and qkv.dim() == 3 and qkv.dtype == torch.bfloat16 and qkv.shape[2] % 3 == 0
            and (qkv.shape[2] // 3) % num_heads == 0
            and native.supports_attention(qkv.shape[1], num_heads, qkv.shape[2] // 3 // num_heads))


def self_attention(qkv: torch.Tensor, num_heads: int) -> torch.Tensor:
    """softmax(Q K^T / sqrt(d)) V per image and head from the packed in-projection output ``qkv`` [N, L, 3C] (head h's
    Q, K, V at columns d*h, C + d*h, 2C + d*h, d = C / num_heads); returns [N, L, C] with head h at columns d*h, the
    input of ``nn.MultiheadAttention``'s out_proj.  Native for bf16 CUDA input with d = 64."""
    if self_attention_native(qkv, num_heads):
        return _SelfAttention.apply(qkv.contiguous(), num_heads)
    return _attention_composite(qkv, num_heads)


# ------------------------------------------------------------------------------------------------
# the encoder block
# ------------------------------------------------------------------------------------------------
class _EncoderBlock(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, num_heads, eps, train, ln1_w, ln1_b, in_w, in_b, out_w, out_b, ln2_w, ln2_b, w1, b1, w2, b2):
        n, L, C = x.shape
        x2 = x.reshape(n * L, C)
        wi, wo, w1b, w2b = weight_bf16(in_w), weight_bf16(out_w), weight_bf16(w1), weight_bf16(w2)
        t1, mean1, rstd1 = native.layer_norm_fwd(x2, ln1_w, ln1_b, eps)
        qkv = _lin(t1, wi, in_b, 3 * C, n)
        o, lse = native.attention_fwd(qkv, num_heads, L)
        a = _lin(o, wo, out_b, C, n)
        x1, t2, mean2, rstd2 = native.add_layer_norm_fwd(x2, a, ln2_w, ln2_b, eps)
        h = _lin(t2, w1b, b1, w1.shape[0], n)
        g = native.gelu_fwd(h)
        y = _lin(g, w2b, b2, C, n)
        z = native.add(x1, y)
        ctx.params = (ln1_w, ln1_b, in_w, in_b, out_w, out_b, ln2_w, ln2_b, w1, b1, w2, b2)
        ctx.dims = (n, L, C, num_heads)
        if train:
            ctx.wb = (wi, wo, w1b, w2b)   # views of the bf16 weight arena: see functional._ConvBnAct
            ctx.save_for_backward(x2, t1, mean1, rstd1, qkv, o, lse, x1, t2, mean2, rstd2, h, g)
        return z.view(n, L, C)

    @staticmethod
    def backward(ctx, dz):
        ln1_w, ln1_b, in_w, in_b, out_w, out_b, ln2_w, ln2_b, w1, b1, w2, b2 = ctx.params
        x2, t1, mean1, rstd1, qkv, o, lse, x1, t2, mean2, rstd2, h, g = ctx.saved_tensors
        wi, wo, w1b, w2b = ctx.wb
        n, L, C, heads = ctx.dims
        dz = dz.contiguous().view(n * L, C)
        if b2.requires_grad:
            native.bias_relu_bwd(dz, dz, grad_buffer(b2), False)
        dg = _dgrad(dz, w2b, w2.shape[1], n)
        _wgrad(w2, g, dz, n)
        dh = native.gelu_bwd(dg, h, _gb(b1))
        dt2 = _dgrad(dh, w1b, C, n)
        _wgrad(w1, t2, dh, n)
        dx1 = native.layer_norm_bwd_add(dt2, x1, mean2, rstd2, ln2_w, dz, _gb(ln2_w), _gb(ln2_b))
        if out_b.requires_grad:
            native.bias_relu_bwd(dx1, dx1, grad_buffer(out_b), False)
        do = _dgrad(dx1, wo, C, n)
        _wgrad(out_w, o, dx1, n)
        dqkv = native.attention_bwd(do, qkv, o, lse, heads, L)
        if in_b.requires_grad:
            native.bias_relu_bwd(dqkv, dqkv, grad_buffer(in_b), False)
        dx = None
        if ctx.needs_input_grad[0] or ln1_w.requires_grad or ln1_b.requires_grad:
            dt1 = _dgrad(dqkv, wi, C, n)
            dx = native.layer_norm_bwd_add(dt1, x2, mean1, rstd1, ln1_w, dx1, _gb(ln1_w), _gb(ln1_b)).view(n, L, C)
        _wgrad(in_w, t1, dqkv, n)
        for p in (b2, w2, b1, w1, ln2_w, ln2_b, out_b, out_w, in_b, in_w, ln1_w, ln1_b):   # LAST, as in _ConvBnAct
            if p.requires_grad:
                notify_ready(p)
        return (dx if ctx.needs_input_grad[0] else None,) + (None,) * 15


def vit_encoder_block_native(x: torch.Tensor, num_heads: int, w1: torch.Tensor) -> bool:
    """Whether :func:`vit_encoder_block` runs on the native node for this input and these weights."""
    if not (use_native(x) and x.dim() == 3 and x.dtype == torch.bfloat16 and x.is_contiguous()):
        return False
    C = x.shape[2]
    return (C % num_heads == 0 and native.supports_attention(x.shape[1], num_heads, C // num_heads)
            and native.supports_layer_norm(C) and native.supports_conv(C, 3 * C)
            and native.supports_conv(C, w1.shape[0]) and native.supports_conv(w1.shape[0], C))


def vit_encoder_block(x: torch.Tensor, num_heads: int, eps: float, ln1_w, ln1_b, in_w, in_b, out_w, out_b, ln2_w,
                      ln2_b, w1, b1, w2, b2) -> torch.Tensor:
    """torchvision's ``EncoderBlock`` (dropout 0) on tokens ``x`` [N, L, C]: x1 = x + MHA(LN1(x)) with the packed
    ``in_w`` [3C, C] / ``in_b`` and ``out_w`` [C, C] / ``out_b``; returns x1 + MLP(LN2(x1)) with ``w1`` [M, C] + ``b1``,
    exact GELU, ``w2`` [C, M] + ``b2``.  Both LayerNorms use ``eps``."""
    params = (ln1_w, ln1_b, in_w, in_b, out_w, out_b, ln2_w, ln2_b, w1, b1, w2, b2)
    if vit_encoder_block_native(x, num_heads, w1):
        train = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        return _EncoderBlock.apply(x, num_heads, eps, train, *params)
    dt = x.dtype if x.is_cuda else ln1_w.dtype
    c = (lambda p: p.to(dt)) if x.is_cuda else (lambda p: p)
    C = x.shape[2]
    t = F.layer_norm(x, (C,), c(ln1_w), c(ln1_b), eps)
    o = _attention_composite(F.linear(t, c(in_w), c(in_b)), num_heads)
    x1 = F.linear(o, c(out_w), c(out_b)) + x
    y = F.layer_norm(x1, (C,), c(ln2_w), c(ln2_b), eps)
    return x1 + F.linear(F.gelu(F.linear(y, c(w1), c(b1))), c(w2), c(b2))


# ------------------------------------------------------------------------------------------------
# patch embedding + class token + position embedding
# ------------------------------------------------------------------------------------------------
class _Embed(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img, weight, bias, cls, pos, patch, train):
        n = img.shape[0]
        rows = native.patchify(img, patch)                                # [N * (L-1), 3 P^2]
        wb = weight_bf16(weight, stem=False)                               # [C, 3 P^2]: KRSC of [C, 3, P, P]
        C = weight.shape[0]
        pe = _lin(rows, wb, bias, C, n)
        tok = native.tokens_fwd(pe, cls.reshape(C), pos.reshape(-1, C), n)
        ctx.params = (weight, bias, cls, pos)
        ctx.n = n
        if train:
            ctx.save_for_backward(rows)
        return tok.view(n, -1, C)

    @staticmethod
    def backward(ctx, dtok):
        weight, bias, cls, pos = ctx.params
        (rows,) = ctx.saved_tensors
        n = ctx.n
        L, C = dtok.shape[1], dtok.shape[2]
        dpe = native.tokens_bwd(dtok.contiguous().view(n * L, C), n, L, _gb(pos), _gb(cls), _gb(bias),
                                want_dpatch=weight.requires_grad)
        if weight.requires_grad:
            _wgrad(weight, rows, dpe, n)
        for p in (pos, cls, bias, weight):
            if p.requires_grad:
                notify_ready(p)
        return (None,) * 7


def vit_embed(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, cls: torch.Tensor, pos: torch.Tensor,
              patch: int) -> torch.Tensor:
    """torchvision's ``VisionTransformer._process_input`` + class token + position embedding: tokens [N, L, C] of the
    image ``x`` with the patch conv ``weight`` [C, 3, P, P] (stride P) + ``bias``, ``cls`` [1, 1, C] and ``pos``
    [1, L, C].  Native for NHWC4 bf16 images (no input gradient: the image is data)."""
    C = weight.shape[0]
    if use_native(x) and x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[1] == 4 \
            and x.is_contiguous(memory_format=torch.channels_last) and (3 * patch * patch) % 64 == 0 \
            and native.supports_conv(3 * patch * patch, C):
        params = (weight, bias, cls, pos)
        train = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        return _Embed.apply(x, weight, bias, cls, pos, patch, train)
    dt = x.dtype if x.is_cuda else weight.dtype
    c = (lambda p: p.to(dt)) if x.is_cuda else (lambda p: p)
    y = F.conv2d(x[:, :3], c(weight), c(bias), stride=patch)
    y = y.reshape(x.shape[0], C, -1).permute(0, 2, 1)
    return torch.cat([c(cls).expand(x.shape[0], -1, -1), y], dim=1) + c(pos)
