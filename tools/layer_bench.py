#!/usr/bin/env python
"""Per-layer kernel timing for the ResNet-50 shapes at batch 256 (CUDA events, L2 flushed between reps).

For every distinct conv of ResNet-50: fwd (+BN-stats epilogue), BN apply, dgrad, wgrad, BN backward —
time, achieved TFLOP/s and GB/s against peak figures (default: NVIDIA's H100 SXM data sheet, 3.35 TB/s HBM3 and 989
dense bf16 TFLOP/s; LB_PEAKS=file.json with {"hbm_gbs", "bf16_tflops"} for measured ones), plus the same conv through
cuDNN (torch, bf16 channels_last) for orientation.  --json PATH also writes the rows as JSON.
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributeddeeplearning_b200.ops import native as nv  # noqa: E402

SHAPES = [  # cin, hw, cout, k, stride, pad, occurrences
    (3, 224, 64, 7, 2, 3, 1), (64, 56, 64, 1, 1, 0, 1), (64, 56, 64, 3, 1, 1, 3), (64, 56, 256, 1, 1, 0, 4),
    (256, 56, 64, 1, 1, 0, 2), (256, 56, 128, 1, 1, 0, 1), (128, 56, 128, 3, 2, 1, 1), (128, 28, 512, 1, 1, 0, 4),
    (256, 56, 512, 1, 2, 0, 1), (512, 28, 128, 1, 1, 0, 3), (128, 28, 128, 3, 1, 1, 3), (512, 28, 256, 1, 1, 0, 1),
    (256, 28, 256, 3, 2, 1, 1), (256, 14, 1024, 1, 1, 0, 6), (512, 28, 1024, 1, 2, 0, 1), (1024, 14, 256, 1, 1, 0, 5),
    (256, 14, 256, 3, 1, 1, 5), (1024, 14, 512, 1, 1, 0, 1), (512, 14, 512, 3, 2, 1, 1), (512, 7, 2048, 1, 1, 0, 3),
    (1024, 14, 2048, 1, 2, 0, 1), (2048, 7, 512, 1, 1, 0, 2), (512, 7, 512, 3, 1, 1, 2),
]


def timeit(fn, reps=5, flush=None):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        if flush is not None:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts)


def main():
    B = int(os.environ.get("LB_BATCH", 256))
    peaks = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}
    if os.environ.get("LB_PEAKS"):
        peaks.update(json.load(open(os.environ["LB_PEAKS"])))
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows = []
    cl = torch.channels_last
    tot = {k: 0.0 for k in ("fwd", "bn", "dgrad", "wgrad", "bnb", "bnbx", "cudnn_fwd", "cudnn_bwd")}
    for (ci, hw, co, k, s, p, occ) in SHAPES:
        P = (hw + 2 * p - k) // s + 1
        if ci == 3:
            x = nv.philox_images(B, hw, hw, 1, 0, dev)
            w = torch.randn(co, 3, k, k, device=dev) * 0.05
            wb = nv.pack_stem_weight(w.contiguous(memory_format=cl), k, k)
            xt = torch.randn(B, 3, hw, hw, device=dev, dtype=torch.bfloat16).contiguous(memory_format=cl)
        else:
            x = torch.randn(B, ci, hw, hw, device=dev, dtype=torch.bfloat16).contiguous(memory_format=cl)
            w = torch.randn(co, ci, k, k, device=dev) * 0.05
            wb = w.permute(0, 2, 3, 1).reshape(co, -1).contiguous().to(torch.bfloat16)
            xt = x
        wt = w.to(torch.bfloat16).contiguous(memory_format=cl)
        y, st = nv.conv_fwd(x, wb, (k, k), s, p, stats=True, cout=co)
        dy = torch.randn_like(y)
        gamma, beta = torch.ones(co, device=dev), torch.zeros(co, device=dev)
        rm, rv = torch.zeros(co, device=dev), torch.ones(co, device=dev)
        gw = torch.zeros(co, ci, k, k, device=dev).contiguous(memory_format=cl)
        z, save = nv.bn_act_fwd(y, st, gamma, beta, rm, rv, 1e-5, 0.1, True, None, True)
        gg, bg = torch.zeros(co, device=dev), torch.zeros(co, device=dev)
        C = nv._C()
        sweep = {}
        # every applicable kernel variant on this shape: time (L2 flushed) + max |difference| against the one-tile
        # kernel's output (the variants share the k order, so their results must agree to bf16 rounding)
        vt = {}
        if ci != 3 and os.environ.get("LB_VARIANTS", "1") == "1":
            M_f, M_d = B * P * P, B * hw * hw
            kb_f = k * k * ((ci + 63) // 64)
            kb_d = k * k * ((co + 63) // 64)
            nt_f, nt_d = (co + 63) // 64 * 64, (ci + 63) // 64 * 64
            for name, cands, run in (
                    ("fwd", nv.conv_variants(nt_f, M_f, kb_f, False),
                     lambda: nv.conv_fwd(x, wb, (k, k), s, p, stats=True, cout=co)[0]),
                    ("dgrad", nv.conv_variants(nt_d, M_d if s == 1 else M_d // 4, kb_d if s == 1 else max(1, kb_d // 4), True),
                     lambda: nv.conv_dgrad(dy, wb, x.shape, (k, k), s, p))):
                ref_out, res = None, {}
                for v in cands:
                    nv.force_variant(v)
                    try:
                        out = run()
                        torch.cuda.synchronize()
                    except RuntimeError as e:
                        res[nv.variant_name(v)] = ("n/a", str(e).splitlines()[0][:40])
                        continue
                    if ref_out is None:
                        ref_out = out.float()
                    diff = float((out.float() - ref_out).abs().max())
                    t_ = timeit(run, reps=3, flush=flush)
                    res[nv.variant_name(v)] = (round(t_ * 1e3, 1), diff)
                nv.force_variant(None)
                vt[name] = res
        sweep["variants_us_maxdiff"] = vt
        f8 = {}
        if os.environ.get("LB_FP8", "0") == "1" and ci % 128 == 0:
            from distributeddeeplearning_b200.ops import fp8 as f8m

            f8m.enable(True)
            nv.conv_fwd(x, wb, (k, k), s, p, stats=True, cout=co)          # calibrate + autotune
            f8["fwd_total"] = timeit(lambda: nv.conv_fwd(x, wb, (k, k), s, p, stats=True, cout=co), flush=flush) * 1e3
            f8["quant_x"] = timeit(lambda: f8m.quantize(x, ("lbx", ci, hw)), flush=flush) * 1e3
            if co % 128 == 0:
                nv.conv_dgrad(dy, wb, x.shape, (k, k), s, p)
                f8["dgrad_total"] = timeit(lambda: nv.conv_dgrad(dy, wb, x.shape, (k, k), s, p), flush=flush) * 1e3
                f8["quant_dy"] = timeit(lambda: f8m.quantize(dy, ("lbdy", co, hw), e5m2=True), flush=flush) * 1e3
            f8m.enable(False)
        sweep["fp8_us"] = {k_: round(v_, 1) for k_, v_ in f8.items()}
        t_fwd = timeit(lambda: nv.conv_fwd(x, wb, (k, k), s, p, stats=True, cout=co), flush=flush)
        t_bn = timeit(lambda: nv.bn_act_fwd(y, st, gamma, beta, rm, rv, 1e-5, 0.1, True, None, True), flush=flush)
        t_dg = timeit(lambda: nv.conv_dgrad(dy, wb, x.shape, (k, k), s, p), flush=flush) if ci != 3 else 0.0
        t_wg = timeit(lambda: nv.conv_wgrad(x, dy, gw, (k, k), s, p), flush=flush)
        t_bnb = timeit(lambda: nv.bn_act_bwd(dy, z, y, save, gamma, True, False, gg, bg), flush=flush)
        t_bnbx = timeit(lambda: nv.bn_act_bwd(dy, z, y, save, gamma, True, False, gg, bg, beta=beta, had_residual=False),
                        flush=flush)
        xr = xt.detach().requires_grad_(ci != 3)
        wr = wt.detach().requires_grad_(True)
        t_cf = timeit(lambda: F.conv2d(xr, wr, None, s, p), flush=flush)
        yy = F.conv2d(xr, wr, None, s, p)
        gy = torch.randn_like(yy)
        t_cb = timeit(lambda: torch.autograd.grad(yy, [wr] + ([xr] if ci != 3 else []), gy, retain_graph=True), flush=flush)
        M = B * P * P
        flops = 2.0 * M * co * ci * k * k
        act_bytes = (B * hw * hw * max(ci, 4) + M * co) * 2
        row = {"shape": f"{ci}x{hw}->{co} k{k}s{s}", "occ": occ, "M": M, "gflop": flops / 1e9,
               "fwd_ms": t_fwd, "fwd_tflops": flops / t_fwd / 1e9, "fwd_gbs": act_bytes / t_fwd / 1e6,
               "bn_ms": t_bn, "bn_gbs": 2 * M * co * 2 / t_bn / 1e6,
               "dgrad_ms": t_dg, "wgrad_ms": t_wg, "bnb_ms": t_bnb, "bnb_maskx_ms": t_bnbx, "stage_sweep": sweep, "bnb_gbs": 4 * M * co * 2 / t_bnb / 1e6,
               "cudnn_fwd_ms": t_cf, "cudnn_bwd_ms": t_cb}
        rows.append(row)
        for key, v in (("fwd", t_fwd), ("bn", t_bn), ("dgrad", t_dg), ("wgrad", t_wg), ("bnb", t_bnb), ("bnbx", t_bnbx),
                       ("cudnn_fwd", t_cf), ("cudnn_bwd", t_cb)):
            tot[key] += v * occ
        print(f"{row['shape']:22s} x{occ} fwd {t_fwd:7.3f}ms {row['fwd_tflops']:7.1f}TF {row['fwd_gbs']:6.0f}GB/s | bn {t_bn:6.3f} "
              f"| dgrad {t_dg:7.3f} | wgrad {t_wg:7.3f} | bnb {t_bnb:6.3f}/{t_bnbx:6.3f} || cudnn fwd {t_cf:7.3f} bwd {t_cb:7.3f}"
              f" || sweep {sweep}", flush=True)
    print("TOTALS (ms, weighted by occurrences):", {k: round(v, 3) for k, v in tot.items()})
    print("ours conv fwd+dgrad+wgrad = %.2f ms, BN fwd+bwd = %.2f ms ; cuDNN conv fwd+bwd = %.2f ms"
          % (tot["fwd"] + tot["dgrad"] + tot["wgrad"], tot["bn"] + tot["bnb"], tot["cudnn_fwd"] + tot["cudnn_bwd"]))
    if "--json" in sys.argv:
        json.dump({"batch": B, "rows": rows, "totals": tot, "peaks": peaks},
                  open(sys.argv[sys.argv.index("--json") + 1], "w"), indent=1)


if __name__ == "__main__":
    main()
