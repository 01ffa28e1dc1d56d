#!/usr/bin/env python
"""Timing of Swin Transformer V2: the scaled-cosine window-attention kernels (csrc/ops/window_attention_v2.cu) at every
stage shape of swin_v2_t and swin_v2_b, at 256 (no padding) and at 224 (stages 2-4 pad to multiples of 8), and the
whole models' training throughput.

Window attention (shift 4 where the padded side exceeds 8) against ``F.scaled_dot_product_attention`` on pre-normalised,
pre-partitioned windows [N, nW * heads, 64, 32] of the padded map, with the logit scale folded into q-hat and the
position bias + shifted-window mask as a float ``attn_mask`` [nW * heads, 64, 64] (normalisation and partition are not
timed).  Forward: O (and the native log-sum-exp); backward: dQ, dK, dV (and the native table, logit-scale and bias
gradients) from dO.  TFLOP/s come from the matrix products of the padded frame at L = 64: forward 4 N nW heads L^2 32
FLOPs, backward 8 N nW heads L^2 32.  CUDA events, L2 flushed before every run, median of --iters runs.

The CPB MLP kernels (forward and backward) at every head count, and their sum over one training step of each model.

Training throughput: ``BenchmarkSession`` (fused allreduce + SGD, CUDA graph) at --batch, at 256 and 224, images/s
over --steps timed steps after warm-up, each configuration in a process of its own.  The card's name, power limit and
maximum SM clock are printed with the tables.

    python tools/swin_v2_bench.py [--batch 256] [--iters 20] [--steps 10] [--models swin_v2_t,swin_v2_b]
                                  [--skip-attention] [--skip-cpb] [--skip-train]
"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from depthwise_bench import card, timed  # noqa: E402

# (model, stage, heads); H = W = size / 4 / 2^(stage - 1), C = 32 heads
STAGES = [("swin_v2_t", 1, 3), ("swin_v2_t", 2, 6), ("swin_v2_t", 3, 12), ("swin_v2_t", 4, 24),
          ("swin_v2_b", 1, 4), ("swin_v2_b", 2, 8), ("swin_v2_b", 3, 16), ("swin_v2_b", 4, 32)]


def _sdpa_inputs(qkv, table, ls, qb, vb, N, H, heads, shift):
    """q-hat * s_h, k-hat, v [N, nW * heads, 64, 32] of the padded, rolled, partitioned map and the float mask
    [nW * heads, 64, 64] (bias + -100 mask)."""
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops.swin import relative_position_index

    C, pH = 32 * heads, -(-H // 8) * 8
    nW = (pH // 8) ** 2
    full = torch.cat([qb, torch.zeros_like(qb), vb]).to(qkv.dtype).expand(N, pH, pH, 3 * C).clone()
    full[:, :H, :H] = qkv.view(N, H, H, 3 * C)
    if shift:
        full = torch.roll(full, (-shift, -shift), (1, 2))
    t = full.view(N, pH // 8, 8, pH // 8, 8, 3, heads, 32).permute(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, N, nW * heads,
                                                                                                  64, 32)
    s = torch.clamp(ls.view(1, heads, 1, 1), max=math.log(100.0)).exp().repeat(1, nW, 1, 1).to(qkv.dtype)
    q = (F.normalize(t[0].float(), dim=-1).to(qkv.dtype) * s).contiguous().requires_grad_(True)
    k = F.normalize(t[1].float(), dim=-1).to(qkv.dtype).contiguous().requires_grad_(True)
    v = t[2].contiguous().requires_grad_(True)
    bias = table[relative_position_index(8).to(qkv.device)].view(64, 64, heads).permute(2, 0, 1)
    reg = torch.zeros(pH, pH, device=qkv.device)
    if shift:
        count = 0
        for h in ((0, -8), (-8, -shift), (-shift, None)):
            for w in ((0, -8), (-8, -shift), (-shift, None)):
                reg[h[0]:h[1], w[0]:w[1]] = count
                count += 1
    reg = reg.view(pH // 8, 8, pH // 8, 8).permute(0, 2, 1, 3).reshape(nW, 64)
    wm = ((reg[:, None, :] - reg[:, :, None]) != 0).float() * -100.0
    mask = (bias[None] + wm[:, None]).reshape(nW * heads, 64, 64).to(torch.bfloat16)
    return q, k, v, mask


def attention_table(a, dev, flush, rows):
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    print(f"# window attention v2 at batch {a.batch}, median of {a.iters} (us); TFLOP/s from the padded frame at L = 64")
    print(f"{'model':>9} {'st':>2} {'HxW':>5} {'h':>2} {'sh':>2} {'pass':>4} | {'native':>8} {'sdpa':>8} | {'TF/s':>6} "
          f"{'TF/s':>6} | {'sdpa/native':>11}")
    for size in (256, 224):
        for model, stage, heads in STAGES:
            N, C, H = a.batch, 32 * heads, size // 4 >> (stage - 1)
            pH = -(-H // 8) * 8
            shift = 4 if pH > 8 else 0
            qkv = torch.randn(N * H * H, 3 * C, device=dev).to(torch.bfloat16)
            table = torch.rand(225, heads, device=dev) * 16
            ls = torch.log(10 * torch.ones(heads, 1, 1, device=dev))
            qb, vb = torch.randn(C, device=dev) * 0.1, torch.randn(C, device=dev) * 0.1
            dout = torch.randn(N * H * H, C, device=dev).to(torch.bfloat16)
            o, lse = nv.window_attention_v2_fwd(qkv, table, ls, qb, vb, heads, N, H, H, shift)
            dt, dls, db = torch.empty(225, heads, device=dev), torch.zeros(heads, device=dev), torch.zeros(3 * C,
                                                                                                          device=dev)
            t_nv = (timed(lambda: nv.window_attention_v2_fwd(qkv, table, ls, qb, vb, heads, N, H, H, shift), a.iters,
                          flush),
                    timed(lambda: nv.window_attention_v2_bwd(dout, qkv, table, ls, qb, vb, o, lse, heads, N, H, H, shift,
                                                             dt, dls, db), a.iters, flush))
            q, k, v, mask = _sdpa_inputs(qkv, table, ls, qb, vb, N, H, heads, shift)

            def s_fwd():
                with torch.no_grad():
                    F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=1.0)

            so = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=1.0)
            dso = torch.randn_like(so)
            t_s = (timed(s_fwd, a.iters, flush),
                   timed(lambda: torch.autograd.grad(so, (q, k, v), dso, retain_graph=True), a.iters, flush))
            del so, q, k, v, mask
            base = N * (pH // 8) ** 2 * heads * 64 * 64 * 32
            for i, (pas, flops) in enumerate((("fwd", 4 * base), ("bwd", 8 * base))):
                tf = [flops / (t[i] * 1e-6) / 1e12 for t in (t_nv, t_s)]
                print(f"{model:>9} {stage:2d} {H:2d}x{H:<2d} {heads:2d} {shift:2d} {pas:>4} | {t_nv[i]:8.1f} "
                      f"{t_s[i]:8.1f} | {tf[0]:6.1f} {tf[1]:6.1f} | {t_s[i] / t_nv[i]:11.2f}")
                rows.append(dict(kind="attention", model=model, size=size, stage=stage, H=H, heads=heads, shift=shift,
                                 batch=N, pass_=pas, native_us=round(t_nv[i], 1), sdpa_us=round(t_s[i], 1),
                                 native_tflops=round(tf[0], 1), sdpa_tflops=round(tf[1], 1)))
            del qkv, dout, o, lse
            torch.cuda.empty_cache()


# (model, blocks per stage, heads per stage)
BLOCKS = {"swin_v2_t": ((2, 2, 6, 2), (3, 6, 12, 24)), "swin_v2_s": ((2, 2, 18, 2), (3, 6, 12, 24)),
          "swin_v2_b": ((2, 2, 18, 2), (4, 8, 16, 32))}


def cpb_table_times(a, dev, flush, rows):
    """The CPB MLP kernels (independent of the batch; forward and backward once per block and step, on the main
    stream) at every head count of the zoo, and their sum over one training step of each model."""
    import torch

    from distributeddeeplearning_b200.ops import native as nv
    from distributeddeeplearning_b200.ops.swin_v2 import relative_coords_table

    print(f"# CPB MLP kernels, median of {a.iters} (us)")
    coords = relative_coords_table(8).to(dev)
    t = {}
    for heads in sorted({h for _, hs in BLOCKS.values() for h in hs}):
        w1, b1 = torch.randn(512, 2, device=dev) * 0.02, torch.zeros(512, device=dev)
        w2 = torch.randn(heads, 512, device=dev) * 0.02
        qkv_b = torch.zeros(96 * heads, device=dev)
        table, _ = nv.cpb_fwd(coords, w1, b1, w2, heads, qkv_b)
        dt = torch.randn_like(table)
        g1, gb, g2 = torch.zeros_like(w1), torch.zeros_like(b1), torch.zeros_like(w2)
        t[heads] = (timed(lambda: nv.cpb_fwd(coords, w1, b1, w2, heads, qkv_b), a.iters, flush),
                    timed(lambda: nv.cpb_bwd(coords, w1, b1, w2, table, dt, heads, g1, gb, g2), a.iters, flush))
        print(f"  heads {heads:2d}: fwd {t[heads][0]:7.1f}  bwd {t[heads][1]:7.1f}")
        rows.append(dict(kind="cpb", heads=heads, fwd_us=round(t[heads][0], 1), bwd_us=round(t[heads][1], 1)))
    for model, (depths, hs) in BLOCKS.items():
        f = sum(d * t[h][0] for d, h in zip(depths, hs))
        b = sum(d * t[h][1] for d, h in zip(depths, hs))
        print(f"  {model}: {sum(depths)} blocks per step, fwd {f:8.1f}  bwd {b:8.1f} us")
        rows.append(dict(kind="cpb_step", model=model, fwd_us=round(f, 1), bwd_us=round(b, 1)))


def train_one(model, size, batch, steps):
    """images/s of one training configuration (run in a process of its own: CUDA-graph pools are not returned)."""
    import torch

    from distributeddeeplearning_b200.parallel import dist
    from distributeddeeplearning_b200.workloads.benchmark import BenchmarkSession, fixed_synthetic_batch

    dist.init()
    torch.manual_seed(0)
    s = BenchmarkSession(model, batch, True, lr=0.01, momentum=0.9)
    s.data, s.target = fixed_synthetic_batch(batch, size, s.num_classes, s.device, seed=17)
    for _ in range(2):
        s.step()
    graph = s.enable_graph(warmup=1)
    for _ in range(2):
        s.step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = s.step()
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / steps
    print(json.dumps(dict(kind="train", model=model, size=size, batch=batch, img_s=round(batch / ms * 1e3, 1),
                          ms_per_step=round(ms, 2), graph=graph, loss_finite=math.isfinite(float(loss)))))


def throughput_table(a, rows):
    import subprocess

    print(f"# training throughput at batch {a.batch} (CUDA graph, fused allreduce + SGD), {a.steps} timed steps")
    for model in a.models.split(","):
        for size in (256, 224):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--train-one", f"{model},{size}", "--batch",
                                str(a.batch), "--steps", str(a.steps)], capture_output=True, text=True)
            lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
            if r.returncode != 0 or not lines:
                print(f"{model:>9} {size:3d}: failed\n{(r.stdout + r.stderr)[-2000:]}", flush=True)
                continue
            row = json.loads(lines[-1])
            print(f"{model:>9} {size:3d}: {row['img_s']:9.1f} img/s  ({row['ms_per_step']:.2f} ms/step, graph "
                  f"{row['graph']}, final loss finite {row['loss_finite']})", flush=True)
            rows.append(row)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--models", default="swin_v2_t,swin_v2_b")
    ap.add_argument("--skip-attention", action="store_true")
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--skip-cpb", action="store_true")
    ap.add_argument("--train-one", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.train_one:
        model, size = a.train_one.split(",")
        return train_one(model, int(size), a.batch, a.steps)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("swin_v2_bench.py needs a GPU")
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    os.environ["DDL_B200_IMPL"] = "native"
    print(f"# {card()} (name, power.limit, clocks.max.sm)")
    rows = []
    if not a.skip_attention:
        attention_table(a, dev, flush, rows)
    if not a.skip_cpb:
        cpb_table_times(a, dev, flush, rows)
    if not a.skip_train:
        throughput_table(a, rows)
    print(json.dumps({"card": card(), "rows": rows}))


if __name__ == "__main__":
    main()
