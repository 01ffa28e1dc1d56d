#!/usr/bin/env python
"""Timing of MaxViT's kernels at the stage shapes of maxvit_t (224: 56/2, 28/4, 14/8, 7/16 map / heads), batch 256,
on the same bf16 operands, and of maxvit_t's training step.

- Grid and window partition attention (csrc/ops/window_attention.cu) against ``F.scaled_dot_product_attention`` on
  pre-partitioned sequences [N, G * heads, 49, 32] with the relative-position bias as a bf16 ``attn_mask`` (the
  partition itself is not timed), and Swin's window kernel at shift 0 (whose scale is 1/sqrt(32), not MaxViT's
  1/sqrt(C): timed for comparison only).  Forward: O (and the native log-sum-exp); backward: dQ, dK, dV (and the native
  bias gradient) from dO.  TFLOP/s from the matrix products at L = 49: forward 4 N G heads L^2 32, backward 8 N G heads
  L^2 32.
- BN-GELU (the fused BN kernels, activation 5) forward and backward against ``F.batch_norm`` + ``F.gelu``, at the
  expanded MBConv widths of each stage.
- maxvit_t training throughput (one-GPU BenchmarkSession with its CUDA graph), at --batch or, when that does not fit,
  the largest of batch / 2, batch / 4, ... that does.

CUDA events, L2 flushed before every kernel run, median of --iters runs; the card's name, power limit and maximum SM
clock are printed with the table.

    python tools/maxvit_bench.py [--batch 256] [--iters 20] [--steps 20]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from depthwise_bench import card, timed  # noqa: E402

# (stage, H = W, heads) of maxvit_t at 224; C = 32 heads
SHAPES = [(1, 56, 2), (2, 28, 4), (3, 14, 8), (4, 7, 16)]


def _sdpa_inputs(qkv, table, N, H, heads, grid):
    """Pre-partitioned q, k, v [N, G * heads, 49, 32] and the bias [G * heads, 49, 49]."""
    import torch

    from distributeddeeplearning_b200.ops import maxvit as mx

    C = 32 * heads
    t = mx._to_seq(qkv.view(N, H, H, 3 * C), grid)                      # [N, G, 49, 3C]
    G = t.shape[1]
    t = t.reshape(N, G, 49, 3, heads, 32).permute(3, 0, 1, 4, 2, 5).reshape(3, N, G * heads, 49, 32)
    q, k, v = (t[i].contiguous().requires_grad_(True) for i in range(3))
    bias = mx.relative_position_bias(table)[0]                            # [heads, 49, 49]
    mask = bias[None].expand(G, heads, 49, 49).reshape(G * heads, 49, 49).to(torch.bfloat16).contiguous()
    return q, k, v, mask


def _train_rate(batch, steps):
    import torch

    from distributeddeeplearning_b200.parallel import dist
    from distributeddeeplearning_b200.workloads.benchmark import BenchmarkSession

    dist.init()
    while batch >= 1:
        try:
            torch.manual_seed(0)
            s = BenchmarkSession("maxvit_t", batch, True, lr=0.01, momentum=0.9)
            for _ in range(3):
                s.step()
            s.enable_graph(warmup=2)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                s.step()
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) / steps
            mem = torch.cuda.max_memory_allocated() / 2 ** 30
            del s
            torch.cuda.empty_cache()
            return batch, batch / dt, dt * 1e3, mem
        except torch.cuda.OutOfMemoryError:
            print(f"# maxvit_t training does not fit at batch {batch}", flush=True)
            torch.cuda.empty_cache()
            batch //= 2
    raise SystemExit("maxvit_t training does not fit at batch 1")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    if not torch.cuda.is_available():
        raise SystemExit("maxvit_bench.py needs a GPU")
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    os.environ["DDL_B200_IMPL"] = "native"
    print(f"# {card()} (name, power.limit, clocks.max.sm); partition attention at batch {a.batch}, median of {a.iters} "
          f"(us); TFLOP/s from the shapes at L = 49 (fwd 4 N G h L^2 32, bwd 8 N G h L^2 32)")
    print(f"{'st':>2} {'HxW':>5} {'h':>2} {'part':>6} {'pass':>4} | {'native':>8} {'sdpa':>8} {'swin win':>8} | "
          f"{'TF/s':>6} {'TF/s':>6}")
    rows = []
    for stage, H, heads in SHAPES:
        N, C = a.batch, 32 * heads
        qkv = torch.randn(N * H * H, 3 * C, device=dev).to(torch.bfloat16)
        table = torch.randn(169, heads, device=dev) * 0.5
        dout = torch.randn(N * H * H, C, device=dev).to(torch.bfloat16)
        dt = torch.zeros(169, heads, device=dev)
        o, lse = nv.window_attention_fwd(qkv, table, heads, N, H, H, 0)
        t_w = (timed(lambda: nv.window_attention_fwd(qkv, table, heads, N, H, H, 0), a.iters, flush),
               timed(lambda: nv.window_attention_bwd(dout, qkv, table, o, lse, heads, N, H, H, 0, dt), a.iters, flush))
        for grid in (True, False):
            sc = C ** -0.5
            o, lse = nv.grid_attention_fwd(qkv, table, heads, N, H, H, sc, grid=grid)
            t_nv = (timed(lambda: nv.grid_attention_fwd(qkv, table, heads, N, H, H, sc, grid=grid), a.iters, flush),
                    timed(lambda: nv.grid_attention_bwd(dout, qkv, table, o, lse, heads, N, H, H, sc, dt, grid=grid),
                          a.iters, flush))
            q, k, v, mask = _sdpa_inputs(qkv, table, N, H, heads, grid)

            def s_fwd():
                with torch.no_grad():
                    F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=sc)

            so = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=sc)
            dso = torch.randn_like(so)
            t_s = (timed(s_fwd, a.iters, flush),
                   timed(lambda: torch.autograd.grad(so, (q, k, v), dso, retain_graph=True), a.iters, flush))
            del so, q, k, v, mask
            base = N * (H // 7) ** 2 * heads * 49 * 49 * 32
            part = "grid" if grid else "window"
            for i, (pas, flops) in enumerate((("fwd", 4 * base), ("bwd", 8 * base))):
                tf = [flops / (t[i] * 1e-6) / 1e12 for t in (t_nv, t_s)]
                print(f"{stage:2d} {H:2d}x{H:<2d} {heads:2d} {part:>6} {pas:>4} | {t_nv[i]:8.1f} {t_s[i]:8.1f} "
                      f"{t_w[i]:8.1f} | {tf[0]:6.1f} {tf[1]:6.1f}")
                rows.append(dict(stage=stage, H=H, heads=heads, partition=part, batch=N, pass_=pas,
                                 native_us=round(t_nv[i], 1), sdpa_us=round(t_s[i], 1),
                                 swin_window_us=round(t_w[i], 1), native_tflops=round(tf[0], 1),
                                 sdpa_tflops=round(tf[1], 1)))
        del qkv, dout, o, lse
        torch.cuda.empty_cache()
    print(f"# BN-GELU (train) at batch {a.batch}, median of {a.iters} (us): native vs F.batch_norm + F.gelu")
    print(f"{'st':>2} {'HxW':>5} {'C':>5} {'pass':>4} | {'native':>8} {'torch':>8}")
    for stage, H, heads in SHAPES:
        C, N = 4 * 32 * heads, a.batch
        y = torch.randn(N, C, H, H, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        g, b = torch.ones(C, device=dev), torch.zeros(C, device=dev)
        rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
        z, save = nv.bn_act_fwd(y, None, g, b, rm, rv, 1e-3, 0.01, 5, None, True)
        dz = torch.randn_like(z)
        gg, bg = torch.zeros_like(g), torch.zeros_like(b)
        t_n = (timed(lambda: nv.bn_act_fwd(y, None, g, b, rm, rv, 1e-3, 0.01, 5, None, True), a.iters, flush),
               timed(lambda: nv.bn_act_bwd(dz, None, y, save, g, 5, False, gg, bg, beta=b, had_residual=False),
                     a.iters, flush))
        yr = y.detach().clone().requires_grad_(True)
        gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)

        def comp():
            return F.gelu(F.batch_norm(yr, rm, rv, gr, br, True, 0.01, 1e-3))

        def comp_fwd():
            with torch.no_grad():
                comp()

        r = comp()
        t_t = (timed(comp_fwd, a.iters, flush),
               timed(lambda: torch.autograd.grad(r, (yr, gr, br), dz, retain_graph=True), a.iters, flush))
        for i, pas in enumerate(("fwd", "bwd")):
            print(f"{stage:2d} {H:2d}x{H:<2d} {C:5d} {pas:>4} | {t_n[i]:8.1f} {t_t[i]:8.1f}")
            rows.append(dict(bn_gelu=True, stage=stage, H=H, C=C, batch=N, pass_=pas, native_us=round(t_n[i], 1),
                             torch_us=round(t_t[i], 1)))
        del y, z, dz, yr, r
        torch.cuda.empty_cache()
    del flush
    torch.cuda.empty_cache()
    bs, rate, ms, mem = _train_rate(a.batch, a.steps)
    print(f"# maxvit_t training (CUDA graph, one GPU): batch {bs}: {rate:.1f} img/s ({ms:.1f} ms/step), "
          f"peak memory {mem:.1f} GiB")
    print(json.dumps({"card": card(), "rows": rows,
                      "train": dict(batch=bs, img_per_s=round(rate, 1), ms_per_step=round(ms, 2),
                                    peak_gib=round(mem, 1))}))


if __name__ == "__main__":
    main()
