#!/usr/bin/env python
"""Per-layer timing of the grouped 3x3 convolutions of ResNeXt-50 32x4d (default) or of one RegNet (``--model
regnet_*``: its distinct grouped layers at 224): native group-bundle kernels (forward with BN statistics, data
gradient, weight gradient, and the per-step weight expansion) against cuDNN's bf16 channels_last grouped convolution
(torch.nn.functional.conv2d and its autograd backward), CUDA events, L2 flushed before every run.

    python tools/grouped_bench.py [--model regnet_y_16gf] [--batch 256] [--iters 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [(128, 56, 1, 4), (256, 56, 2, 8), (256, 28, 1, 8), (512, 28, 2, 16), (512, 14, 1, 16), (1024, 14, 2, 32),
          (1024, 7, 1, 32)]


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--model", default=None, help="a regnet_* name: time its grouped layers instead of ResNeXt-50's")
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.models import regnet
    from distributeddeeplearning_b200.ops import native as nv

    if a.model is not None and a.model not in regnet._PARAMS:
        ap.error(f"--model must be one of {sorted(regnet._PARAMS)}")
    shapes = SHAPES if a.model is None else regnet.grouped_shapes(a.model)

    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    print(f"# {torch.cuda.get_device_name(0)}, {a.model or 'resnext50_32x4d'}, batch {a.batch}, median of {a.iters} (us)")
    print(f"{'C':>5} {'HW':>3} {'s':>1} {'cg':>3} | {'fwd':>8} {'cudnn':>8} | {'dgrad':>8} {'cudnn':>8} | {'wgrad':>8} "
          f"{'cudnn':>8} | {'expand':>6}")
    rows = []
    for C, hw, s, cg in shapes:
        g = C // cg
        x = torch.randn(a.batch, C, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(C, cg, 3, 3, device=dev) * 0.1).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        wc = w.permute(0, 2, 3, 1).reshape(C, 9 * cg).contiguous()
        we = nv.expand_grouped_weight(wc, 9, g)
        y = nv.conv_fwd(x, we, (3, 3), s, 1, stats=True, groups=g)[0]
        dy = torch.randn_like(y)
        gw = torch.zeros(C, cg, 3, 3, device=dev).contiguous(memory_format=torch.channels_last)
        r = {"C": C, "HW": hw, "stride": s, "cg": cg}
        r["fwd"] = timed(lambda: nv.conv_fwd(x, we, (3, 3), s, 1, stats=True, groups=g), a.iters, flush)
        r["fwd_cudnn"] = timed(lambda: F.conv2d(x, w, None, s, 1, 1, g), a.iters, flush)
        r["dgrad"] = timed(lambda: nv.conv_dgrad(dy, we, x.shape, (3, 3), s, 1, groups=g), a.iters, flush)
        r["dgrad_cudnn"] = timed(lambda: torch.ops.aten.convolution_backward(
            dy, x, w, None, [s, s], [1, 1], [1, 1], False, [0, 0], g, [True, False, False]), a.iters, flush)
        r["wgrad"] = timed(lambda: nv.conv_wgrad(x, dy, gw, (3, 3), s, 1, groups=g), a.iters, flush)
        r["wgrad_cudnn"] = timed(lambda: torch.ops.aten.convolution_backward(
            dy, x, w, None, [s, s], [1, 1], [1, 1], False, [0, 0], g, [False, True, False]), a.iters, flush)
        r["expand"] = timed(lambda: nv.expand_grouped_weight(wc, 9, g), a.iters, flush)
        rows.append(r)
        print(f"{C:5d} {hw:3d} {s:1d} {cg:3d} | {r['fwd']:8.1f} {r['fwd_cudnn']:8.1f} | {r['dgrad']:8.1f} "
              f"{r['dgrad_cudnn']:8.1f} | {r['wgrad']:8.1f} {r['wgrad_cudnn']:8.1f} | {r['expand']:6.1f}", flush=True)
    tot = {k: sum(r[k] for r in rows) for k in ("fwd", "fwd_cudnn", "dgrad", "dgrad_cudnn", "wgrad", "wgrad_cudnn")}
    print("total  " + "  ".join(f"{k}={v:.0f}" for k, v in tot.items()))
    print("JSON " + json.dumps({"device": torch.cuda.get_device_name(0), "model": a.model or "resnext50_32x4d",
                                "batch": a.batch, "rows": rows}))


if __name__ == "__main__":
    sys.exit(main())
