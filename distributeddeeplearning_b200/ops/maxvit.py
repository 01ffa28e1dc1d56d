"""MaxViT ops: grid attention, torchvision's ``PartitionAttentionLayer`` as ONE autograd node (the Swin block's node
with the partition-attention kernels), stochastic depth + residual for MBConv, and tanh on [B, F].

    attention layer (dropout 0), on the NHWC rows [N*H*W, C] in image order:
      t1 = LN1(x);  qkv = t1 Wqkv^T + bqkv;  o = pattn(qkv);  a = o Wm^T + bm;  x1 = x + keep1[n] * a
      t2 = LN2(x1);  y = fc2(gelu(fc1(t2)));  z = x1 + keep2[n] * y

torchvision partitions the map first and runs every op on the partitioned tensor.  LayerNorm, the linears and the
per-sample stochastic depth act on one token at a time, so they commute with the partition: the native node runs them on
the image-order rows and the attention kernels (csrc/ops/window_attention.cu) gather each sequence from qkv with index
arithmetic.  The window partition puts token t = 7a + b of sequence (i, j) at pixel (7i + a, 7j + b), the grid partition
(WindowPartition(H/7) + SwapAxes) at (a H/7 + i, b H/7 + j).

torchvision's ``RelativePositionalMultiHeadAttention`` scales k by ``feat_dim ** -0.5``, feat_dim being the layer's
channel count C, not the head dim: the logits are q . k / sqrt(C).  The composites of torch ops are exactly
torchvision's maths; they are the CPU path and the float64 oracle of the tests.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from . import native
from .functional import CL, use_native
from .swin import _SwinBlock, _ones, swin_block_native

PARTITION = 7


# ------------------------------------------------------------------------------------------------
# composites (torchvision's maths)
# ------------------------------------------------------------------------------------------------
def _partition(t: torch.Tensor, p: int) -> torch.Tensor:
    """torchvision's ``WindowPartition`` on an NHWC map [B, H, W, c]: [B, (H/p)(W/p), p*p, c]."""
    B, H, W, c = t.shape
    return t.reshape(B, H // p, p, W // p, p, c).permute(0, 1, 3, 2, 4, 5).reshape(B, (H // p) * (W // p), p * p, c)


def _departition(t: torch.Tensor, p: int, H: int, W: int) -> torch.Tensor:
    """torchvision's ``WindowDepartition`` back to an NHWC map [B, H, W, c]."""
    B, c = t.shape[0], t.shape[-1]
    return t.reshape(B, H // p, W // p, p, p, c).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, c)


def _to_seq(t: torch.Tensor, grid: bool) -> torch.Tensor:
    """NHWC map -> [B, G, 49, c] sequences of the window (p = 7) or grid (p = H/7, then SwapAxes(-2, -3)) partition."""
    if grid:
        return _partition(t, t.shape[1] // PARTITION).transpose(1, 2)
    return _partition(t, PARTITION)


def _from_seq(t: torch.Tensor, grid: bool, H: int, W: int) -> torch.Tensor:
    if grid:
        return _departition(t.transpose(1, 2), H // PARTITION, H, W)
    return _departition(t, PARTITION, H, W)


def relative_position_bias(table: torch.Tensor) -> torch.Tensor:
    """torchvision's ``get_relative_positional_bias``: [1, heads, 49, 49] from the table [169, heads]."""
    from .swin import relative_position_index

    idx = relative_position_index(PARTITION).to(table.device)
    return table[idx].view(49, 49, -1).permute(2, 0, 1).contiguous().unsqueeze(0)


def _attend(seq: torch.Tensor, table: torch.Tensor, heads: int) -> torch.Tensor:
    """torchvision's RelativePositionalMultiHeadAttention without ``merge`` on qkv sequences [B, G, P, 3C]."""
    B, G, P, c3 = seq.shape
    C = c3 // 3
    q, k, v = torch.chunk(seq, 3, dim=-1)
    q = q.reshape(B, G, P, heads, C // heads).permute(0, 1, 3, 2, 4)
    k = k.reshape(B, G, P, heads, C // heads).permute(0, 1, 3, 2, 4)
    v = v.reshape(B, G, P, heads, C // heads).permute(0, 1, 3, 2, 4)
    k = k * C ** -0.5
    a = torch.einsum("B G H I D, B G H J D -> B G H I J", q, k)
    a = F.softmax(a + relative_position_bias(table).to(a.dtype), dim=-1)
    o = torch.einsum("B G H I J, B G H J D -> B G H I D", a, v)
    return o.permute(0, 1, 3, 2, 4).reshape(B, G, P, C)


def _attend_map(qkv: torch.Tensor, table: torch.Tensor, heads: int, grid: bool) -> torch.Tensor:
    """Partition attention on an NHWC qkv map [B, H, W, 3C] -> [B, H, W, C]."""
    H, W = qkv.shape[1], qkv.shape[2]
    return _from_seq(_attend(_to_seq(qkv, grid), table, heads), grid, H, W)


# ------------------------------------------------------------------------------------------------
# the attention functional
# ------------------------------------------------------------------------------------------------
class _GridAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, table, heads, N, H, W):
        scale = (qkv.shape[1] // 3) ** -0.5
        o, lse = native.grid_attention_fwd(qkv, table, heads, N, H, W, scale)
        ctx.save_for_backward(qkv, table, o, lse)
        ctx.dims = (heads, N, H, W, scale)
        return o

    @staticmethod
    def backward(ctx, do):
        qkv, table, o, lse = ctx.saved_tensors
        heads, N, H, W, scale = ctx.dims
        dtable = torch.zeros_like(table) if ctx.needs_input_grad[1] else None
        dqkv = native.grid_attention_bwd(do.contiguous(), qkv, table, o, lse, heads, N, H, W, scale, dtable)
        return dqkv, dtable, None, None, None, None


def grid_attention_native(qkv: torch.Tensor, heads: int, H: int, W: int) -> bool:
    """Whether :func:`grid_attention` runs on the native kernels for this input."""
    return (use_native(qkv) and qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.shape[1] % 3 == 0
            and (qkv.shape[1] // 3) % heads == 0
            and native.supports_grid_attention(H, W, PARTITION, heads, qkv.shape[1] // 3 // heads))


def grid_attention(qkv: torch.Tensor, table: torch.Tensor, heads: int, H: int, W: int) -> torch.Tensor:
    """MaxViT's grid attention from the qkv rows [N*H*W, 3C] of a square NHWC map in image order (head h's Q, K, V at
    columns d h, C + d h, 2C + d h) with the relative-position bias ``table`` [169, heads]: token t = 7a + b of sequence
    (i, j) is pixel (a H/7 + i, b H/7 + j), and the logits are q . k / sqrt(C) + bias (torchvision's scale).  Returns the
    attention output rows [N*H*W, C] in image order, the input of ``merge``.  Native for bf16 CUDA input with head
    dim 32 and H = W a multiple of 7."""
    N = qkv.shape[0] // (H * W)
    if grid_attention_native(qkv, heads, H, W):
        return _GridAttention.apply(qkv.contiguous(), table, heads, N, H, W)
    c3 = qkv.shape[1]
    o = _attend_map(qkv.reshape(N, H, W, c3), table.to(qkv.dtype) if qkv.is_cuda else table, heads, True)
    return o.reshape(N * H * W, c3 // 3)


# ------------------------------------------------------------------------------------------------
# the attention layer
# ------------------------------------------------------------------------------------------------
def maxvit_attention_layer_native(x: torch.Tensor, heads: int, w1: torch.Tensor) -> bool:
    """Whether :func:`maxvit_attention_layer` runs on the native node for this input and these weights."""
    if not (use_native(x) and x.dim() == 4 and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=CL)):
        return False
    N, C, H, W = x.shape
    return (C % heads == 0 and native.supports_grid_attention(H, W, PARTITION, heads, C // heads)
            and swin_block_native(x, heads, PARTITION, w1))


def maxvit_attention_layer(x: torch.Tensor, partition: str, heads: int, eps: float, n1_w, n1_b, qkv_w, qkv_b, merge_w,
                           merge_b, table, n2_w, n2_b, w1, b1, w2, b2, keep1: Optional[torch.Tensor] = None,
                           keep2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torchvision's ``PartitionAttentionLayer`` (dropout 0) on the NHWC activation ``x`` [N, C, H, W] with
    ``partition`` "window" or "grid": x1 = x + keep1[n] * merge(pattn(qkv(LN1(x)))) with the relative-position bias
    ``table`` [169, heads] and logits scaled by 1/sqrt(C); returns x1 + keep2[n] * fc2(gelu(fc1(LN2(x1)))).
    ``keep1`` / ``keep2``: independent fp32 [N] stochastic-depth scales (``stochastic_depth_keep``), or None."""
    if partition not in ("window", "grid"):
        raise ValueError(f"maxvit_attention_layer: partition must be 'window' or 'grid', got {partition!r}")
    grid = partition == "grid"
    params = (n1_w, n1_b, qkv_w, qkv_b, merge_w, merge_b, table, n2_w, n2_b, w1, b1, w2, b2)
    N, C, H, W = x.shape
    if maxvit_attention_layer_native(x, heads, w1):
        train = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
        return _SwinBlock.apply(x, keep1, keep2, heads, 0, (grid, C ** -0.5), eps, train, *params)
    dt = x.dtype if x.is_cuda else n1_w.dtype
    c = (lambda p: p.to(dt)) if x.is_cuda else (lambda p: p)
    xs = x.permute(0, 2, 3, 1)
    qkv = F.linear(F.layer_norm(xs, (C,), c(n1_w), c(n1_b), eps), c(qkv_w), c(qkv_b))
    a = F.linear(_attend_map(qkv, c(table), heads, grid), c(merge_w), c(merge_b))
    if keep1 is not None:
        a = a * keep1.to(a.dtype).view(-1, 1, 1, 1)
    x1 = xs + a
    y = F.linear(F.gelu(F.linear(F.layer_norm(x1, (C,), c(n2_w), c(n2_b), eps), c(w1), c(b1))), c(w2), c(b2))
    if keep2 is not None:
        y = y * keep2.to(y.dtype).view(-1, 1, 1, 1)
    z = (x1 + y).permute(0, 3, 1, 2)
    return z.contiguous(memory_format=CL) if x.is_cuda else z


# ------------------------------------------------------------------------------------------------
# MBConv's stochastic depth + residual, and tanh
# ------------------------------------------------------------------------------------------------
class _StochasticDepthAdd(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, res, keep):
        ctx.keep = keep
        if keep is None:
            return native.add(y, res)
        return native.layer_scale_fwd(y, _ones(y.shape[1], y.device), keep, res)

    @staticmethod
    def backward(ctx, dz):
        if not dz.is_contiguous(memory_format=CL):
            dz = dz.contiguous(memory_format=CL)
        if ctx.keep is None:
            return dz, dz, None
        # y is only read for the layer-scale gradient, which is not wanted: dz stands in for it
        dy = native.layer_scale_bwd(dz, dz, _ones(dz.shape[1], dz.device), ctx.keep, None, None)
        return dy, dz, None


def stochastic_depth_add(y: torch.Tensor, res: torch.Tensor, keep: Optional[torch.Tensor] = None) -> torch.Tensor:
    """res + keep[n] * y for NHWC activations (MBConv's residual; ``keep``: stochastic-depth scales, or None): one kernel
    in each direction on the native path."""
    if use_native(y) and y.dtype == torch.bfloat16 and y.shape == res.shape and y.shape[1] % 8 == 0 \
            and y.is_contiguous(memory_format=CL) and res.is_contiguous(memory_format=CL):
        return _StochasticDepthAdd.apply(y, res, keep)
    return res + (y if keep is None else y * keep.to(y.dtype).view(-1, 1, 1, 1))


class _Tanh(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y = native.tanh_rows_fwd(x)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        return native.tanh_rows_bwd(dy.contiguous(), y)


def tanh(x: torch.Tensor) -> torch.Tensor:
    """tanh(x); the native backward is dy * (1 - y^2) from the saved output."""
    if use_native(x) and x.dtype == torch.bfloat16 and x.is_contiguous() and x.numel() % 8 == 0:
        return _Tanh.apply(x)
    return torch.tanh(x)
