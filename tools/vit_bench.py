#!/usr/bin/env python
"""Timing of the fused multi-head self-attention kernels (csrc/ops/attention.cu) at the ViT layer shapes, batch 256,
against ``F.scaled_dot_product_attention`` restricted to torch's flash backend, on the same bf16 operands.

The native kernels read Q, K and V out of the packed in-projection output [N*L, 3C] and write O as [N*L, C]; torch gets
strided [N, H, L, 64] views of the same qkv buffer.  Forward: O and the log-sum-exp; backward: dQ, dK, dV from dO (the
native backward is its dQ kernel plus its dK/dV kernel).  CUDA events, L2 flushed before every run, median of --iters
runs.  TFLOP/s come from the matrix products the algorithm needs, computed from the shapes and the same for both
implementations: forward 2 products (Q K^T, P V) = 4 N H L^2 64 FLOPs, backward 4 (dV, dP, dQ, dK) = 8 N H L^2 64
(recomputation of S inside a backward is not counted).  The card's name, power limit and maximum SM clock are printed
with the table.

    python tools/vit_bench.py [--batch 256] [--iters 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from depthwise_bench import card, timed  # noqa: E402

# (label, tokens L, hidden C): ViT-B/16 and -B/32 (C 768, 12 heads), ViT-L/16 and -L/32 (C 1024, 16 heads) at 224
SHAPES = [("vit_b_16", 197, 768), ("vit_b_32", 50, 768), ("vit_l_16", 197, 1024), ("vit_l_32", 50, 1024)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from distributeddeeplearning_b200.ops import native as nv

    if not torch.cuda.is_available():
        raise SystemExit("vit_bench.py needs a GPU")
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    print(f"# {card()} (name, power.limit, clocks.max.sm); attention at batch {a.batch}, median of {a.iters} (us); "
          f"TFLOP/s from the shapes (fwd 4 N H L^2 d, bwd 8 N H L^2 d)")
    print(f"{'shape':>9} {'L':>4} {'C':>5} {'pass':>4} | {'native':>8} {'flash':>8} | {'TF/s':>6} {'TF/s':>6}")
    rows = []
    for label, L, C in SHAPES:
        N, H = a.batch, C // 64
        qkv = torch.randn(N * L, 3 * C, device=dev).to(torch.bfloat16)
        dout = torch.randn(N * L, C, device=dev).to(torch.bfloat16)
        o, lse = nv.attention_fwd(qkv, H, L)
        v3 = qkv.view(N, L, 3, H, 64)
        q, k, v = (v3[:, :, i].transpose(1, 2).detach().requires_grad_(True) for i in range(3))
        do4 = dout.view(N, L, H, 64).transpose(1, 2)
        with sdpa_kernel([SDPBackend.FLASH_ATTENTION]):
            ref = F.scaled_dot_product_attention(q, k, v)
            err = float((ref.detach().transpose(1, 2).reshape(N * L, C).float() - o.float()).abs().max())

            def t_fwd():
                with torch.no_grad():
                    F.scaled_dot_product_attention(q, k, v)

            def t_bwd():
                torch.autograd.grad(ref, (q, k, v), do4, retain_graph=True)

            times_ref = (timed(t_fwd, a.iters, flush), timed(t_bwd, a.iters, flush))
        times_nv = (timed(lambda: nv.attention_fwd(qkv, H, L), a.iters, flush),
                    timed(lambda: nv.attention_bwd(dout, qkv, o, lse, H, L), a.iters, flush))
        base = N * H * L * L * 64
        for pas, flops, tn, tr in (("fwd", 4 * base, times_nv[0], times_ref[0]), ("bwd", 8 * base, times_nv[1], times_ref[1])):
            tfn, tfr = flops / (tn * 1e-6) / 1e12, flops / (tr * 1e-6) / 1e12
            print(f"{label:>9} {L:4d} {C:5d} {pas:>4} | {tn:8.1f} {tr:8.1f} | {tfn:6.1f} {tfr:6.1f}")
            rows.append(dict(shape=label, L=L, C=C, heads=H, batch=N, pass_=pas, native_us=round(tn, 1),
                             flash_us=round(tr, 1), native_tflops=round(tfn, 1), flash_tflops=round(tfr, 1)))
        print(f"#   {label}: max |O native - O flash| = {err:.3e}")
    print(json.dumps({"card": card(), "rows": rows}))


if __name__ == "__main__":
    main()
