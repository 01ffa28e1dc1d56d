#!/usr/bin/env python
"""Timing of the shifted-window attention kernels (csrc/ops/window_attention.cu) and of patch merge + LayerNorm
(csrc/ops/swin.cu) at the stage shapes of swin_t and swin_b, batch 256, on the same bf16 operands.

Window attention (shift 3 on stages 1-3; stage 4 is one window, shift 0) against
- torchvision's composite (pad, roll, partition, bias + mask, softmax, reverse, roll back: ``ops.window_attention``'s
  torch path) on the image-order qkv rows, and
- ``F.scaled_dot_product_attention`` on pre-partitioned windows [N, nW * heads, 49, 32] with the relative-position
  bias + shifted-window mask as a float ``attn_mask`` [nW * heads, 49, 49] (the partition itself is not timed).
Forward: O (and the native log-sum-exp); backward: dQ, dK, dV (and the native bias gradient) from dO.  TFLOP/s come
from the matrix products at L = 49: forward 4 N nW heads L^2 32 FLOPs, backward 8 N nW heads L^2 32.
Patch merge + LN (forward, and backward with dgamma / dbeta) against torch's gather + ``F.layer_norm``.
CUDA events, L2 flushed before every run, median of --iters runs; the card's name, power limit and maximum SM clock
are printed with the table.

    python tools/swin_bench.py [--batch 256] [--iters 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from depthwise_bench import card, timed  # noqa: E402

# (model, stage, H = W, heads); C = 32 heads
SHAPES = [("swin_t", 1, 56, 3), ("swin_t", 2, 28, 6), ("swin_t", 3, 14, 12), ("swin_t", 4, 7, 24),
          ("swin_b", 1, 56, 4), ("swin_b", 2, 28, 8), ("swin_b", 3, 14, 16), ("swin_b", 4, 7, 32)]
# (model, merge, H = W of the input, C of the input)
MERGES = [("swin_t", 1, 56, 96), ("swin_t", 2, 28, 192), ("swin_t", 3, 14, 384),
          ("swin_b", 1, 56, 128), ("swin_b", 2, 28, 256), ("swin_b", 3, 14, 512)]


def _sdpa_inputs(qkv, table, N, H, heads, shift):
    """Pre-partitioned q, k, v [N, nW * heads, 49, 32] and the float mask [nW * heads, 49, 49] (bias + -100 mask)."""
    import torch

    from distributeddeeplearning_b200.ops.swin import relative_position_index

    C, nW = 32 * heads, (H // 7) ** 2
    t = qkv.view(N, H, H, 3 * C)
    if shift:
        t = torch.roll(t, (-shift, -shift), (1, 2))
    t = t.view(N, H // 7, 7, H // 7, 7, 3, heads, 32).permute(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, N, nW * heads, 49, 32)
    q, k, v = (t[i].contiguous().requires_grad_(True) for i in range(3))
    bias = table[relative_position_index(7).to(qkv.device)].view(49, 49, heads).permute(2, 0, 1)
    reg = torch.zeros(H, H, device=qkv.device)
    if shift:
        count = 0
        for h in ((0, -7), (-7, -shift), (-shift, None)):
            for w in ((0, -7), (-7, -shift), (-shift, None)):
                reg[h[0]:h[1], w[0]:w[1]] = count
                count += 1
    reg = reg.view(H // 7, 7, H // 7, 7).permute(0, 2, 1, 3).reshape(nW, 49)
    wm = ((reg[:, None, :] - reg[:, :, None]) != 0).float() * -100.0
    mask = (bias[None] + wm[:, None]).reshape(nW * heads, 49, 49).to(torch.bfloat16)
    return q, k, v, mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv
    from distributeddeeplearning_b200.ops import swin

    if not torch.cuda.is_available():
        raise SystemExit("swin_bench.py needs a GPU")
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    os.environ["DDL_B200_IMPL"] = "native"
    print(f"# {card()} (name, power.limit, clocks.max.sm); window attention at batch {a.batch}, median of {a.iters} "
          f"(us); TFLOP/s from the shapes at L = 49 (fwd 4 N nW h L^2 32, bwd 8 N nW h L^2 32)")
    print(f"{'model':>6} {'st':>2} {'HxW':>5} {'h':>2} {'sh':>2} {'pass':>4} | {'native':>8} {'tv comp':>8} {'sdpa':>8} | "
          f"{'TF/s':>6} {'TF/s':>6} {'TF/s':>6}")
    rows = []
    for model, stage, H, heads in SHAPES:
        N, C, shift = a.batch, 32 * heads, 3 if H > 7 else 0
        qkv = torch.randn(N * H * H, 3 * C, device=dev).to(torch.bfloat16)
        table = torch.randn(169, heads, device=dev) * 0.5
        dout = torch.randn(N * H * H, C, device=dev).to(torch.bfloat16)
        o, lse = nv.window_attention_fwd(qkv, table, heads, N, H, H, shift)
        dt = torch.zeros(169, heads, device=dev)
        t_nv = (timed(lambda: nv.window_attention_fwd(qkv, table, heads, N, H, H, shift), a.iters, flush),
                timed(lambda: nv.window_attention_bwd(dout, qkv, table, o, lse, heads, N, H, H, shift, dt), a.iters,
                      flush))
        # torchvision's composite (the torch path of ops.window_attention) on the same bf16 rows
        qc = qkv.detach().clone().requires_grad_(True)
        tc_ = table.detach().clone().requires_grad_(True)
        os.environ["DDL_B200_IMPL"] = "torch"
        try:
            def c_fwd():
                with torch.no_grad():
                    swin.window_attention(qc, tc_, heads, H, H, 7, shift)

            ref = swin.window_attention(qc, tc_, heads, H, H, 7, shift)
            err = float((ref.detach().float() - o.float()).abs().max())
            t_c = (timed(c_fwd, a.iters, flush),
                   timed(lambda: torch.autograd.grad(ref, (qc, tc_), dout, retain_graph=True), a.iters, flush))
        finally:
            os.environ["DDL_B200_IMPL"] = "native"
        del ref
        q, k, v, mask = _sdpa_inputs(qkv, table, N, H, heads, shift)

        def s_fwd():
            with torch.no_grad():
                F.scaled_dot_product_attention(q, k, v, attn_mask=mask)

        so = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        dso = torch.randn_like(so)
        t_s = (timed(s_fwd, a.iters, flush),
               timed(lambda: torch.autograd.grad(so, (q, k, v), dso, retain_graph=True), a.iters, flush))
        del so, q, k, v, mask
        base = N * (H // 7) ** 2 * heads * 49 * 49 * 32
        for i, (pas, flops) in enumerate((("fwd", 4 * base), ("bwd", 8 * base))):
            tf = [flops / (t[i] * 1e-6) / 1e12 for t in (t_nv, t_c, t_s)]
            print(f"{model:>6} {stage:2d} {H:2d}x{H:<2d} {heads:2d} {shift:2d} {pas:>4} | {t_nv[i]:8.1f} {t_c[i]:8.1f} "
                  f"{t_s[i]:8.1f} | {tf[0]:6.1f} {tf[1]:6.1f} {tf[2]:6.1f}")
            rows.append(dict(model=model, stage=stage, H=H, heads=heads, shift=shift, batch=N, pass_=pas,
                             native_us=round(t_nv[i], 1), composite_us=round(t_c[i], 1), sdpa_us=round(t_s[i], 1),
                             native_tflops=round(tf[0], 1), composite_tflops=round(tf[1], 1),
                             sdpa_tflops=round(tf[2], 1)))
        print(f"#   {model} stage {stage}: max |O native - O composite| = {err:.3e}")
        del qkv, dout, o, lse, qc
        torch.cuda.empty_cache()
    print(f"# patch merge + LayerNorm at batch {a.batch}, median of {a.iters} (us)")
    print(f"{'model':>6} {'m':>2} {'HxW':>5} {'4C':>5} {'pass':>4} | {'native':>8} {'torch':>8}")
    for model, mi, H, C in MERGES:
        N = a.batch
        x = torch.randn(N, C, H, H, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        g, b = torch.ones(4 * C, device=dev), torch.zeros(4 * C, device=dev)
        y, mean, rstd = nv.patch_merge_fwd(x, g, b, 1e-5)
        dy = torch.randn_like(y)
        dg, db = torch.zeros_like(g), torch.zeros_like(b)
        t_n = (timed(lambda: nv.patch_merge_fwd(x, g, b, 1e-5), a.iters, flush),
               timed(lambda: nv.patch_merge_bwd(dy, x, mean, rstd, g, dg, db), a.iters, flush))
        xr = x.detach().clone().requires_grad_(True)
        gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)

        def comp():
            t = xr.permute(0, 2, 3, 1)
            t = torch.cat([t[:, 0::2, 0::2], t[:, 1::2, 0::2], t[:, 0::2, 1::2], t[:, 1::2, 1::2]], -1)
            return F.layer_norm(t, (4 * C,), gr.to(t.dtype), br.to(t.dtype), 1e-5)

        def comp_fwd():
            with torch.no_grad():
                comp()

        r = comp()
        dyr = dy.view_as(r)
        t_t = (timed(comp_fwd, a.iters, flush),
               timed(lambda: torch.autograd.grad(r, (xr, gr, br), dyr, retain_graph=True), a.iters, flush))
        for i, pas in enumerate(("fwd", "bwd")):
            print(f"{model:>6} {mi:2d} {H:2d}x{H:<2d} {4 * C:5d} {pas:>4} | {t_n[i]:8.1f} {t_t[i]:8.1f}")
            rows.append(dict(model=model, merge=mi, H=H, C4=4 * C, batch=N, pass_=pas, native_us=round(t_n[i], 1),
                             torch_us=round(t_t[i], 1)))
        del x, y, dy, xr, r
        torch.cuda.empty_cache()
    print(json.dumps({"card": card(), "rows": rows}))


if __name__ == "__main__":
    main()
