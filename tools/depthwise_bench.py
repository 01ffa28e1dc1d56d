#!/usr/bin/env python
"""Per-layer timing of the depthwise convolutions of MobileNetV2 (3x3), MobileNetV3-Large / -Small or EfficientNet-B0
(3x3 and 5x5), or ConvNeXt-Tiny (7x7 with a bias):
native stencil kernels (forward with BN statistics, data gradient, weight gradient) against cuDNN's bf16 channels_last
F.conv2d(groups=C) and aten.convolution_backward.  CUDA events, L2 flushed before every run, median of --iters runs.
For 7x7 the forward adds the bias (cuDNN's too), the weight gradient also reduces the bias gradient, and the forward and
data gradient are timed twice: with the shared-memory halo tile the model uses, and with the L1 mapping of the 5x5
kernels (columns fwd-L1, dgrad-L1), the comparison that decides which of the two the model keeps.

A depthwise convolution is bound by HBM bandwidth, so each row also gives the achieved bandwidth from the bytes the pass must
move (forward: read x, write y; data gradient: read dy, write dx; weight gradient: read x and dy) and its fraction of
the H100 SXM data sheet's 3.35 TB/s.  The card's name, power limit and maximum SM clock are printed with the table.

    python tools/depthwise_bench.py [--model mobilenet_v2|mobilenet_v3_large|mobilenet_v3_small|efficientnet_b0|
                                             convnext_tiny]
                                    [--batch 256]
                                    [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (C, H=W of the input, stride, layers of MobileNetV2 with this shape)
SHAPES = [(32, 112, 1, 1), (96, 112, 2, 1), (144, 56, 1, 1), (144, 56, 2, 1), (192, 28, 1, 2), (192, 28, 2, 1),
          (384, 14, 1, 4), (576, 14, 1, 2), (576, 14, 2, 1), (960, 7, 1, 3)]
# (C, H=W of the input, kernel, stride, layers with this shape) of MobileNetV3
SHAPES_V3 = {
    "mobilenet_v3_large": [(16, 112, 3, 1, 1), (64, 112, 3, 2, 1), (72, 56, 3, 1, 1), (72, 56, 5, 2, 1),
                           (120, 28, 5, 1, 2), (240, 28, 3, 2, 1), (200, 14, 3, 1, 1), (184, 14, 3, 1, 2),
                           (480, 14, 3, 1, 1), (672, 14, 3, 1, 1), (672, 14, 5, 2, 1), (960, 7, 5, 1, 2)],
    "mobilenet_v3_small": [(16, 112, 3, 2, 1), (72, 56, 3, 2, 1), (88, 28, 3, 1, 1), (96, 28, 5, 2, 1),
                           (240, 14, 5, 1, 2), (120, 14, 5, 1, 1), (144, 14, 5, 1, 1), (288, 14, 5, 2, 1),
                           (576, 7, 5, 1, 2)],
    "efficientnet_b0": [(32, 112, 3, 1, 1), (96, 112, 3, 2, 1), (144, 56, 3, 1, 1), (144, 56, 5, 2, 1),
                        (240, 28, 5, 1, 1), (240, 28, 3, 2, 1), (480, 14, 3, 1, 2), (480, 14, 5, 1, 1),
                        (672, 14, 5, 1, 2), (672, 14, 5, 2, 1), (1152, 7, 5, 1, 3), (1152, 7, 3, 1, 1)],
    "convnext_tiny": [(96, 56, 7, 1, 3), (192, 28, 7, 1, 3), (384, 14, 7, 1, 9), (768, 7, 7, 1, 3)],
}
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def timed(fn, iters, flush):
    import torch

    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()                         # evict the operands from L2 (50 MB on H100; 256 MB buffer)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--model", default="mobilenet_v2", choices=["mobilenet_v2", *SHAPES_V3])
    a = ap.parse_args()
    v3 = a.model != "mobilenet_v2"
    shapes = SHAPES_V3[a.model] if v3 else [(C, hw, 3, s, n) for C, hw, s, n in SHAPES]
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    if not torch.cuda.is_available():
        raise SystemExit("depthwise_bench.py needs a GPU")
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    info = card()
    print(f"# {info} (name, power.limit, clocks.max.sm); batch {a.batch}, median of {a.iters} (us); GB/s from the "
          f"bytes each pass must move; % of {HBM_BYTES_PER_S / 1e12:.2f} TB/s (bandwidth-bound)")
    if v3:
        print(f"# {a.model}")
    print(f"{'C':>4} {'HW':>3} " + (f"{'k':>1} " if v3 else "") + f"{'s':>1} {'n':>1} | {'fwd':>7} {'cudnn':>7} {'GB/s':>5} {'%':>3} | {'dgrad':>7} {'cudnn':>7} "
          f"{'GB/s':>5} {'%':>3} | {'wgrad':>7} {'cudnn':>7} {'GB/s':>5} {'%':>3}"
          + (f" | {'fwd-L1':>7} {'dgrad-L1':>8}" if a.model == "convnext_tiny" else ""))
    rows = []
    for C, hw, k, s, n in shapes:
        p = k // 2
        x = torch.randn(a.batch, C, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(C, 1, k, k, device=dev) * 0.3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        wb = w.reshape(C, k * k).contiguous()
        b = torch.randn(C, device=dev)
        y = nv.dwconv7_fwd(x, wb, b) if k == 7 else nv.dwconv_fwd(x, wb, s, k=k)
        dy = torch.randn_like(y)
        gw = torch.zeros(C, 1, k, k, device=dev).contiguous(memory_format=torch.channels_last)
        gb = torch.zeros(C, device=dev)
        bx, by = x.numel() * 2, y.numel() * 2
        r = {"C": C, "HW": hw, **({"k": k} if v3 else {}), "stride": s, "layers": n, "bytes_fwd": bx + by,
             "bytes_dgrad": by + bx, "bytes_wgrad": bx + by}
        if k == 7:
            r["fwd"] = timed(lambda: nv.dwconv7_fwd(x, wb, b), a.iters, flush)
            r["fwd_L1"] = timed(lambda: nv.dwconv7_fwd(x, wb, b, l1=True), a.iters, flush)
            r["fwd_cudnn"] = timed(lambda: F.conv2d(x, w, b.to(torch.bfloat16), s, p, 1, C), a.iters, flush)
            r["dgrad"] = timed(lambda: nv.dwconv7_dgrad(dy, wb), a.iters, flush)
            r["dgrad_L1"] = timed(lambda: nv.dwconv7_dgrad(dy, wb, l1=True), a.iters, flush)
            r["wgrad"] = timed(lambda: nv.dwconv7_wgrad(x, dy, gw, gb), a.iters, flush)
        else:
            r["fwd"] = timed(lambda: nv.dwconv_fwd(x, wb, s, stats=True, k=k), a.iters, flush)
            r["fwd_cudnn"] = timed(lambda: F.conv2d(x, w, None, s, p, 1, C), a.iters, flush)
            r["dgrad"] = timed(lambda: nv.dwconv_dgrad(dy, wb, x.shape, s, k=k), a.iters, flush)
            r["wgrad"] = timed(lambda: nv.dwconv_wgrad(x, dy, gw, s, k=k), a.iters, flush)
        r["dgrad_cudnn"] = timed(lambda: torch.ops.aten.convolution_backward(
            dy, x, w, None, [s, s], [p, p], [1, 1], False, [0, 0], C, [True, False, False]), a.iters, flush)
        r["wgrad_cudnn"] = timed(lambda: torch.ops.aten.convolution_backward(
            dy, x, w, None, [s, s], [p, p], [1, 1], False, [0, 0], C, [False, True, False]), a.iters, flush)
        cells = []
        for ph in ("fwd", "dgrad", "wgrad"):
            gbs = r[f"bytes_{ph}"] / (r[ph] * 1e-6) / 1e9
            r[f"{ph}_GBps"] = gbs
            r[f"{ph}_frac_peak"] = gbs * 1e9 / HBM_BYTES_PER_S
            cells.append(f"{r[ph]:7.1f} {r[ph + '_cudnn']:7.1f} {gbs:5.0f} {100 * r[ph + '_frac_peak']:3.0f}")
        if k == 7:
            cells.append(f"{r['fwd_L1']:7.1f} {r['dgrad_L1']:8.1f}")
        rows.append(r)
        print(f"{C:4d} {hw:3d} " + (f"{k:1d} " if v3 else "") + f"{s:1d} {n:1d} | " + " | ".join(cells), flush=True)
    tot = {k: sum(r[k] * r["layers"] for r in rows)
           for k in ("fwd", "fwd_cudnn", "dgrad", "dgrad_cudnn", "wgrad", "wgrad_cudnn", "fwd_L1", "dgrad_L1")
           if k in rows[0]}
    print(f"all {sum(r['layers'] for r in rows)} layers (us): " + "  ".join(f"{k}={v:.0f}" for k, v in tot.items()))
    print("JSON " + json.dumps({"device": info, "batch": a.batch, **({"model": a.model} if v3 else {}), "rows": rows,
                                "totals_us": tot}))


if __name__ == "__main__":
    sys.exit(main())
