#!/usr/bin/env python
"""GPU kernel diagnostics: every native kernel vs a plain PyTorch fp32 reference of the same op.

Each group runs in its own subprocess with a timeout, so a trap / illegal address / hang in one
kernel cannot take the others (or the GPU box) down.  Prints one line per check:
    [ok|FAIL] name  max_abs=..  rel=..
Usage:  python tools/gpu_diag.py            (all groups)      python tools/gpu_diag.py --group conv_fwd
"""
import argparse
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

GROUPS = ["fp8", "benchshape", "elementwise", "zoo", "graph", "zoograd", "gemm", "conv_generic", "conv_fwd", "conv_dgrad", "conv_wgrad", "linear", "bn", "sgd", "model"]
RESULTS = []


def report(name, got, ref, tol=2e-2, atol=None):
    import torch

    got, ref = got.float(), ref.float()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-12
    rel = err / scale
    ok = (rel <= tol) if atol is None else (err <= atol + tol * scale)
    bad = not torch.isfinite(got).all().item()
    ok = ok and not bad
    print(f"[{'ok' if ok else 'FAIL'}] {name:58s} max_abs={err:.4e} rel={rel:.3e}" + (" NONFINITE" if bad else ""), flush=True)
    RESULTS.append(ok)
    return ok


def cl(t):
    import torch

    return t.contiguous(memory_format=torch.channels_last)


def bf(t):
    import torch

    return t.to(torch.bfloat16)


def report_abs(name, got, ref, rtol, atol):
    """allclose-style check: |got - ref| <= atol + rtol * |ref| ELEMENT-WISE (small-magnitude errors are not hidden
    behind max|ref| the way `report` normalises)."""
    import torch

    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    bound = atol + rtol * ref.abs()
    bad = int((err > bound).sum().item())
    worst = float((err / bound).max().item())
    ok = bad == 0 and bool(torch.isfinite(got).all().item())
    print(f"[{'ok' if ok else 'FAIL'}] {name:58s} violations={bad}/{err.numel()} worst={worst:.3f}x of (atol {atol:g} + rtol {rtol:g}*|ref|)",
          flush=True)
    RESULTS.append(ok)
    return ok


def g_fp8():
    """FP8 operand path: quantisation kernels vs torch.float8 casts; e4m3 x e4m3 forward and e5m2 x e4m3 data-gradient
    convolutions (fp8 wgmma, one-tile kernel) vs an fp32 convolution of the DE-QUANTISED operands (isolates
    the kernel from the quantisation error) and vs the unquantised fp32 result (bounds the quantisation error)."""
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import fp8
    from distributeddeeplearning_b200.ops import native as nv

    dev = torch.device("cuda")
    fp8.reset()
    fp8.enable(True)
    fp8.MIN_K = 0          # kernel correctness on every geometry; the K >= 512 policy is a speed choice
    # ---- quantise: codes must equal torch's float8 cast of x * scale, scale must be a power of two covering amax
    for e5m2, tdt, fmax in ((False, torch.float8_e4m3fn, 448.0), (True, torch.float8_e5m2, 57344.0)):
        x = cl(bf(torch.randn(4, 128, 9, 9, device=dev) * 3.7))
        q, idx = fp8.quantize(x, ("t", e5m2), e5m2=e5m2)
        torch.cuda.synchronize()
        slot = fp8._table(dev)[idx].tolist()
        scale = slot[1]
        amax = float(x.float().abs().max())
        ok = scale > 0 and abs(scale * slot[2] - 1.0) < 1e-6 and (scale * amax <= fmax) and (2 * scale * amax > fmax)
        import math
        ok = ok and abs(math.log2(scale) - round(math.log2(scale))) < 1e-6
        print(f"[{'ok' if ok else 'FAIL'}] fp8 slot e5m2={e5m2}: amax={amax:.3f} scale={scale:g} inv={slot[2]:g}")
        RESULTS.append(ok)
        ref = (x.float() * scale).clamp(-fmax, fmax).to(tdt).view(torch.uint8)
        same = (q.reshape(-1) == ref.reshape(-1)).float().mean().item()
        print(f"[{'ok' if same > 0.999 else 'FAIL'}] fp8 codes e5m2={e5m2}: {same * 100:.3f}% identical to torch cast")
        RESULTS.append(same > 0.999)
    # ---- forward convs (n, cin, h, w, cout, k, stride, pad): M >= one wave of 128-row tiles
    for (n, ci, h, w_, co, k, s, p) in [(32, 128, 28, 28, 256, 1, 1, 0), (32, 256, 28, 28, 128, 3, 1, 1),
                                        (32, 128, 56, 56, 128, 3, 2, 1), (40, 512, 28, 28, 1024, 1, 2, 0),
                                        (32, 256, 28, 28, 64, 1, 1, 0), (128, 512, 14, 14, 512, 3, 1, 1)]:
        x = cl(bf(torch.randn(n, ci, h, w_, device=dev).relu() * 1.5))
        w = bf(torch.randn(co, ci, k, k, device=dev) * (1.0 / (ci * k * k) ** 0.5))
        wb = _w_bf16(w)
        before = fp8.launches()["fwd"]
        y, st = nv.conv_fwd(x, wb, (k, k), s, p, stats=True)
        torch.cuda.synchronize()
        assert fp8.launches()["fwd"] == before + 1, "fp8 forward path not taken"
        xq, sx = fp8.quantize(x, ("x", wb.data_ptr(), n, h, w_))
        wq, sw = fp8.quantize_weight(wb)
        tab = fp8._table(dev)
        xd = xq.view(torch.float8_e4m3fn).float() * tab[sx, 2]
        wd = (wq.view(torch.float8_e4m3fn).float() * tab[sw, 2]).view(co, k, k, ci).permute(0, 3, 1, 2)
        ref_q = F.conv2d(xd, wd, None, s, p)
        report(f"fp8 conv_fwd n{n} c{ci} {h}x{w_}->{co} k{k}s{s} vs dequantised", y, ref_q, 1e-2)
        report("  vs unquantised fp32", y, _conv_ref(x, w, s, p), 8e-2)
        report("  stats sum", st[0], y.float().sum((0, 2, 3)), 2e-3, atol=1e-1)
        fp8.end_of_step()
    # ---- data gradients
    for (n, ci, h, w_, co, k, s, p) in [(32, 128, 28, 28, 256, 1, 1, 0), (32, 256, 28, 28, 128, 3, 1, 1),
                                        (32, 128, 56, 56, 128, 3, 2, 1), (32, 256, 56, 56, 512, 1, 2, 0),
                                        (128, 512, 14, 14, 512, 3, 1, 1)]:
        w = bf(torch.randn(co, ci, k, k, device=dev) * (1.0 / (ci * k * k) ** 0.5))
        wb = _w_bf16(w)
        P = (h + 2 * p - k) // s + 1
        dy = cl(bf(torch.randn(n, co, P, P, device=dev) * 1e-3))
        xs = (n, ci, h, w_)
        before = fp8.launches()["dgrad"]
        dx = nv.conv_dgrad(dy, wb, xs, (k, k), s, p)
        torch.cuda.synchronize()
        assert fp8.launches()["dgrad"] == before + 1, "fp8 dgrad path not taken"
        dq, sd = fp8.quantize(dy, ("dy", wb.data_ptr(), n, P, P), e5m2=True)
        wq, sw = fp8.quantize_weight(wb)
        tab = fp8._table(dev)
        dd = dq.view(torch.float8_e5m2).float() * tab[sd, 2]
        wd = (wq.view(torch.float8_e4m3fn).float() * tab[sw, 2]).view(co, k, k, ci).permute(0, 3, 1, 2)
        ref_q = torch.nn.grad.conv2d_input(xs, wd, dd, s, p)
        report(f"fp8 conv_dgrad n{n} c{ci} {h}x{w_}<-{co} k{k}s{s} vs dequantised", dx, ref_q, 1e-2)
        ref = torch.nn.grad.conv2d_input(xs, w.float(), dy.float(), s, p)
        report("  vs unquantised fp32", dx, ref, 1.5e-1)
        fp8.end_of_step()
    # ---- producer-side twins: BN-apply forward (e4m3) and BN backward (e5m2) emit the fp8 copy in their own pass
    ch, n, hw = 256, 16, 14
    yb = cl(bf(torch.randn(n, ch, hw, hw, device=dev) * 2 + 0.3))
    gamma, beta = torch.rand(ch, device=dev) + 0.5, torch.randn(ch, device=dev) * 0.1
    rm, rv = torch.zeros(ch, device=dev), torch.ones(ch, device=dev)
    for attempt in ("calibrating call", "fused call"):
        fp8._WANTED.update({("act", gamma.data_ptr(), n, hw, hw), ("grad", gamma.data_ptr(), n, hw, hw)})
        z, save = nv.bn_act_fwd(yb, None, gamma, beta, rm, rv, 1e-5, 0.1, True, None, True)
        tw = fp8.twin_of(z)
        assert tw is not None, "bn_act_fwd produced no fp8 twin"
        zq, idx = tw
        torch.cuda.synchronize()
        sc = float(fp8._table(dev)[idx, 1])
        # the fused kernel rounds the fp32 value once to e4m3 (the calibrating call rounds the bf16 tensor): compare the
        # de-quantised twin with z at e4m3 resolution (3 mantissa bits: relative step 2^-3, half of it after rounding)
        deq = zq.view(torch.float8_e4m3fn).float() / sc
        report_abs(f"BN-apply e4m3 twin ({attempt}), scale {sc:g}", deq, z.float(), 0.0725, 2e-3 / sc * 64)
        dz = cl(bf(torch.randn_like(z.float()) * 1e-3))
        dy, _, _ = nv.bn_act_bwd(dz, z, yb, save, gamma, True, False, torch.zeros(ch, device=dev), torch.zeros(ch, device=dev),
                                 beta=beta, had_residual=False)
        tw = fp8.twin_of(dy)
        assert tw is not None, "bn_act_bwd produced no fp8 twin"
        dq, idx = tw
        torch.cuda.synchronize()
        sc = float(fp8._table(dev)[idx, 1])
        deq = dq.view(torch.float8_e5m2).float() / sc
        report(f"BN-backward e5m2 twin ({attempt}) vs bf16 dy, scale {sc:g}", deq, dy.float(), 0.14)
        fp8.end_of_step()
    fp8.enable(False)


def g_benchshape():
    """Benchmark-shape cases (batch 256 layer1 / layer4 of ResNet-50; M = 802,816 and 12,544 rows) through EVERY
    kernel variant the autotuner can pick, checked element-wise (atol + rtol*|ref|) against fp32."""
    import torch

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    for (n, ci, hw, co, k, s, p) in [(256, 64, 56, 64, 3, 1, 1), (256, 64, 56, 256, 1, 1, 0), (256, 512, 7, 512, 3, 1, 1),
                                     (256, 2048, 7, 512, 1, 1, 0), (256, 256, 14, 256, 3, 1, 1)]:
        x = cl(bf(torch.randn(n, ci, hw, hw, device=dev)))
        w = bf(torch.randn(co, ci, k, k, device=dev) * (1.0 / (ci * k * k) ** 0.5))
        wb = _w_bf16(w)
        ref = _conv_ref(x, w, s, p)
        P = (hw + 2 * p - k) // s + 1
        dy = cl(bf(torch.randn(n, co, P, P, device=dev)))
        ref_dx = torch.nn.grad.conv2d_input(x.shape, w.float(), dy.float(), s, p)
        kb = k * k * ((ci + 63) // 64)
        for v in nv.conv_variants((co + 63) // 64 * 64, n * P * P, kb, False):
            nv.force_variant(v)
            y, st = nv.conv_fwd(x, wb, (k, k), s, p, stats=True)
            report_abs(f"fwd {ci}x{hw}->{co} k{k} [{nv.variant_name(v)}]", y, ref, 1.6e-2, 2e-2)
            report("  stats sum", st[0], y.float().sum((0, 2, 3)), 2e-3, atol=2.0)
        for v in nv.conv_variants((ci + 63) // 64 * 64, n * hw * hw, k * k * ((co + 63) // 64), True):
            nv.force_variant(v)
            dx = nv.conv_dgrad(dy, wb, x.shape, (k, k), s, p)
            report_abs(f"dgrad {ci}x{hw}<-{co} k{k} [{nv.variant_name(v)}]", dx, ref_dx, 1.6e-2, 3e-2)
        nv.force_variant(None)


# ------------------------------------------------------------------------------------------------
def g_elementwise():
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    x = nv.philox_images(8, 64, 64, 7, 0, torch.device(dev))
    xf = x.float()
    print(f"philox: mean={xf[:, :3].mean().item():.4f} std={xf[:, :3].std().item():.4f} pad_max={xf[:, 3].abs().max().item()}")
    RESULTS.append(abs(xf[:, :3].mean().item()) < 0.02 and abs(xf[:, :3].std().item() - 1) < 0.02 and xf[:, 3].abs().max().item() == 0)
    lab = nv.philox_labels(4096, 1000, 3, 0, torch.device(dev))
    RESULTS.append(int(lab.min()) >= 0 and int(lab.max()) < 1000 and lab.float().std().item() > 200)
    print(f"labels: min={int(lab.min())} max={int(lab.max())} std={lab.float().std().item():.1f}")
    # softmax xent (padded logits)
    B, Cn, ld = 64, 1000, 1024
    lg = torch.randn(B, ld, device=dev) * 3
    lg[:, Cn:] = 0
    lgb = bf(lg)
    y = torch.randint(0, Cn, (B,), device=dev)
    loss, dl, corr = nv.softmax_xent(lgb[:, :Cn], y, Cn, True, None, True)
    ref = lgb[:, :Cn].float().requires_grad_(True)
    rl = F.cross_entropy(ref, y)
    rl.backward()
    report("softmax_xent loss", loss.reshape(1), rl.detach().reshape(1), 1e-3)
    report("softmax_xent dlogits", dl, ref.grad, 2e-2)
    top = ref.detach().topk(5, 1)[1]
    r1, r5 = (top[:, 0] == y).sum().item(), (top == y[:, None]).sum().item()
    print(f"topk: got {corr.tolist()} ref {[r1, r5]}")
    RESULTS.append(corr.tolist() == [r1, r5])
    # pools
    x = cl(bf(torch.randn(4, 64, 17, 17, device=dev)))
    for (k, s, p) in [(3, 2, 1), (2, 2, 0), (3, 2, 0)]:
        yk, arg = nv.maxpool_fwd(x, k, s, p)
        xr = x.float().requires_grad_(True)
        yr = F.max_pool2d(xr, k, s, p)
        report(f"maxpool fwd k{k}s{s}p{p}", yk, yr.detach(), 1e-6)
        dy = cl(bf(torch.randn_like(yr)))
        yr.backward(dy.float())
        report(f"maxpool bwd k{k}s{s}p{p}", nv.maxpool_bwd(dy, arg, x.shape, k, s, p), xr.grad, 1e-2)
    # even image, 3x3 / s2 / p1: the 2x2-patch specialisation (ResNet stem geometry)
    for (n_, c_, h_, w_) in [(2, 64, 16, 12), (3, 24, 112, 112)]:
        xe = cl(bf(torch.randn(n_, c_, h_, w_, device=dev)))
        yk, arg = nv.maxpool_fwd(xe, 3, 2, 1)
        xr = xe.float().requires_grad_(True)
        yr = F.max_pool2d(xr, 3, 2, 1)
        dy = cl(bf(torch.randn_like(yr)))
        yr.backward(dy.float())
        report(f"maxpool bwd k3s2p1 even {h_}x{w_} c{c_}", nv.maxpool_bwd(dy, arg, xe.shape, 3, 2, 1), xr.grad, 1e-2)
    for cip in (True, False):
        ya = nv.avgpool_fwd(x, 3, 1, 1, cip)
        xr = x.float().contiguous().requires_grad_(True)      # NCHW-contiguous oracle (torch's channels_last
        yr = F.avg_pool2d(xr, 3, 1, 1, count_include_pad=cip)  # avg_pool2d backward mis-handles strided grads)
        report(f"avgpool fwd cip={cip}", ya, yr.detach(), 1e-2)
        dy = cl(bf(torch.randn_like(yr)))
        yr.backward(dy.float().contiguous())
        report(f"avgpool bwd cip={cip}", nv.avgpool_bwd(dy, x.shape, 3, 1, 1, cip), xr.grad, 1e-2)
    g = nv.global_avgpool_fwd(x)
    report("global_avgpool fwd", g, x.float().mean((2, 3)), 1e-2)
    dg = bf(torch.randn(4, 64, device=dev))
    report("global_avgpool bwd", nv.global_avgpool_bwd(dg, x.shape), (dg.float() / 289)[:, :, None, None].expand(4, 64, 17, 17), 1e-2)
    # conversions
    img = torch.rand(3, 3, 20, 24, device=dev)
    mean, std = torch.tensor([0.485, 0.456, 0.406], device=dev), torch.tensor([0.229, 0.224, 0.225], device=dev)
    o = nv.nchw_to_nhwc4(img, mean, std)
    report("nchw_to_nhwc4", o[:, :3], (img - mean.view(1, 3, 1, 1)) / std.view(1, 3, 1, 1), 1e-2)
    u8 = torch.randint(0, 256, (3, 21, 23, 3), dtype=torch.uint8, device=dev)
    o = nv.u8_nhwc_to_nhwc4(u8, mean, std)
    refu = ((u8.float() / 255 - mean) / std).permute(0, 3, 1, 2)
    report("u8_nhwc_to_nhwc4", o[:, :3], refu, 1e-2)
    RESULTS.append(o[:, 3].abs().max().item() == 0)
    a, b = bf(torch.randn(4096, device=dev)), bf(torch.randn(4096, device=dev))
    report("add", nv.add(a, b), a.float() + b.float(), 1e-2)
    d = nv.dropout(bf(torch.ones(1 << 16, device=dev)), 0.5, 1, 0)
    keep = (d != 0).float().mean().item()
    print(f"dropout keep={keep:.4f} scale={d.max().item()}")
    RESULTS.append(abs(keep - 0.5) < 0.02 and d.max().item() == 2.0)
    # device-resident step counter (CUDA-graph replays): same step -> same mask, next step -> a fresh mask
    ones = bf(torch.ones(1 << 16, device=dev))
    step = torch.zeros((), dtype=torch.int64, device=dev)
    m0, m0b = nv.dropout(ones, 0.5, 1, 0, step), nv.dropout(ones, 0.5, 1, 0, step)
    step.add_(1)
    m1 = nv.dropout(ones, 0.5, 1, 0, step)
    same, frac = bool((m0 == m0b).all()), float((m0 != m1).float().mean())
    print(f"dropout step counter: repeatable={same} changed fraction after advance={frac:.3f}")
    RESULTS.append(same and 0.4 < frac < 0.6)
    dz, z = cl(bf(torch.randn(2, 192, 5, 5, device=dev))), cl(bf(torch.randn(2, 192, 5, 5, device=dev)))
    db = torch.zeros(192, device=dev)
    dx = nv.bias_relu_bwd(dz, z, db, True)
    refdx = dz.float() * (z.float() > 0)
    report("bias_relu_bwd dx", dx, refdx, 1e-6)
    report("bias_relu_bwd dbias", db, refdx.sum((0, 2, 3)), 1e-3)


def _conv_ref(x, w, stride, pad, dil=1):
    import torch
    import torch.nn.functional as F

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return F.conv2d(x.float(), w.float(), None, stride, pad, dil)


def _w_bf16(w):
    # logical [Cout,Cin,R,S] -> KRSC matrix [Cout, R*S*Cin] bf16
    return bf(w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous())


def g_gemm():
    import torch

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    for (M, K, N) in [(128, 64, 64), (256, 128, 128), (300, 256, 192), (1000, 512, 256), (4099, 64, 128)]:
        hw = 1
        x = cl(bf(torch.randn(M, K, 1, 1, device=dev)))
        w = bf(torch.randn(N, K, 1, 1, device=dev) * 0.1)
        y, st = nv.conv_fwd(x, _w_bf16(w), (1, 1), 1, 0, stats=True)
        ref = _conv_ref(x, w, 1, 0)
        report(f"gemm(1x1 TMA-A) M{M} K{K} N{N}", y, ref, 2e-2)
        yb = y.float()
        report(f"  stats sum  M{M} K{K} N{N}", st[0], yb.sum((0, 2, 3)), 2e-3, atol=1e-2)
        report(f"  stats sumsq M{M} K{K} N{N}", st[1], (yb * yb).sum((0, 2, 3)), 2e-3)


def g_conv_fwd():
    import torch

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    cases = [(2, 64, 56, 56, 128, 3, 2, 1), (3, 256, 14, 14, 512, 1, 2, 0), (2, 128, 13, 13, 128, 3, 2, 1), (3, 64, 7, 7, 64, 3, 1, 1), (5, 128, 14, 14, 128, 3, 1, 1), (2, 64, 56, 56, 128, 3, 1, 1), (2, 64, 28, 28, 64, 3, 1, 1), (2, 64, 15, 15, 64, 3, 1, 0), (1, 64, 20, 20, 64, 3, 1, 2), (2, 64, 8, 8, 64, 3, 1, 1), (2, 64, 9, 9, 128, 3, 2, 1), (3, 128, 14, 14, 128, 3, 1, 1),
             (2, 256, 7, 7, 512, 1, 2, 0), (2, 64, 12, 12, 192, 5, 1, 2), (1, 192, 13, 13, 384, 3, 1, 1),
             (4, 64, 56, 56, 64, 3, 1, 1)]
    for (n, ci, h, w_, co, k, s, p) in cases:
        x = cl(bf(torch.randn(n, ci, h, w_, device=dev)))
        w = bf(torch.randn(co, ci, k, k, device=dev) * (1.0 / (ci * k * k) ** 0.5))
        y, st = nv.conv_fwd(x, _w_bf16(w), (k, k), s, p, stats=True)
        ref = _conv_ref(x, w, s, p)
        report(f"conv_fwd n{n} c{ci} {h}x{w_} ->{co} k{k}s{s}p{p}", y, ref, 2e-2)
        report("  stats sum", st[0], y.float().sum((0, 2, 3)), 2e-3, atol=1e-2)
    # bias + relu epilogue
    x = cl(bf(torch.randn(2, 64, 10, 10, device=dev)))
    w = bf(torch.randn(128, 64, 3, 3, device=dev) * 0.05)
    b = torch.randn(128, device=dev)
    y = nv.conv_fwd(x, _w_bf16(w), (3, 3), 1, 1, bias=b, relu=True)
    report("conv_fwd bias+relu", y, torch.relu(_conv_ref(x, w, 1, 1) + b.view(1, -1, 1, 1)), 2e-2)
    # stems: ResNet 7x7/2, AlexNet 11x11/4, VGG 3x3/1
    for tma in (True, False):       # TMA-fed (row-interleaved padded image) and cp.async gather stems
        nv.USE_STEM_TMA = tma
        for (k, s, p, hw) in [(7, 2, 3, 32), (11, 4, 2, 63), (3, 1, 1, 16), (3, 2, 0, 35), (7, 2, 0, 41), (7, 2, 3, 224)]:
            img = torch.randn(2, 3, hw, hw, device=dev)
            x4 = nv.nchw_to_nhwc4(img)
            w = torch.randn(64, 3, k, k, device=dev) * 0.1
            wp = nv.pack_stem_weight(cl(w), k, k)
            y, st = nv.conv_fwd(x4, wp, (k, k), s, p, stats=True, cout=64)
            ref = _conv_ref(bf(img), bf(w), s, p)
            report(f"stem conv {'tma' if tma else 'gather'} k{k}s{s}p{p} {hw}x{hw}", y, ref, 2e-2)
    nv.USE_STEM_TMA = True


def g_conv_generic():
    """Channel counts that are not multiples of 64, rectangular kernels, asymmetric padding — fwd / dgrad / wgrad through
    the TMA tile path and (DDL_DISABLE_TILE_TMA-style) the cp.async gather path, plus BN on odd widths."""
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    # n, cin, h, w, cout, (R, S), stride, (ph, pw)
    cases = [(2, 32, 17, 17, 48, (3, 3), 1, (1, 1)), (2, 48, 17, 17, 64, (5, 5), 1, (2, 2)),
             (2, 80, 15, 15, 192, (3, 3), 1, (0, 0)), (2, 160, 17, 17, 160, (1, 7), 1, (0, 3)),
             (2, 160, 17, 17, 192, (7, 1), 1, (3, 0)), (2, 288, 17, 17, 384, (3, 3), 2, (0, 0)),
             (2, 96, 16, 16, 96, (3, 3), 2, (0, 0)), (3, 192, 9, 9, 320, (1, 1), 1, (0, 0)),
             (2, 448, 8, 8, 384, (3, 3), 1, (1, 1)), (2, 24, 12, 12, 40, (3, 3), 1, (1, 1)),
             (2, 384, 8, 8, 384, (1, 3), 1, (0, 1)), (2, 32, 20, 20, 32, (3, 3), 3, (1, 1)),
             (2, 1280, 8, 8, 320, (1, 1), 1, (0, 0)), (2, 64, 16, 16, 96, (1, 1), 2, (0, 0))]
    for tile in (True, False):
        nv.USE_TILE_TMA = tile
        for (n, ci, h, w_, co, k, s, p) in cases:
            x = torch.randn(n, ci, h, w_, device=dev).to(torch.bfloat16).float().requires_grad_(True)
            w = bf(torch.randn(co, ci, k[0], k[1], device=dev) * (1.0 / (ci * k[0] * k[1]) ** 0.5)).float().requires_grad_(True)
            ref = F.conv2d(x, w, None, s, p)
            dy = cl(bf(torch.randn_like(ref)))
            ref.backward(dy.float())
            xb = cl(x.detach().to(torch.bfloat16))
            wb = w.detach().permute(0, 2, 3, 1).reshape(co, -1).contiguous().to(torch.bfloat16)
            tag = f"{'tile' if tile else 'gather'} n{n} c{ci} {h}x{w_} ->{co} k{k[0]}x{k[1]} s{s} p{p}"
            y, st = nv.conv_fwd(xb, wb, k, s, p, stats=True)
            report(f"fwd   {tag}", y, ref, 2e-2)
            report("   stats sum", st[0], y.float().sum((0, 2, 3)), 2e-3, atol=2e-2)
            report("   stats sumsq", st[1], (y.float() ** 2).sum((0, 2, 3)), 2e-3, atol=2e-2)
            dx = nv.conv_dgrad(dy, wb, x.shape, k, s, p)
            report(f"dgrad {tag}", dx, x.grad, 2e-2)
            gw = cl(torch.zeros(co, ci, k[0], k[1], device=dev))
            nv.conv_wgrad(xb, dy, gw, k, s, p)
            report(f"wgrad {tag}", gw, w.grad, 2e-2)
    nv.USE_TILE_TMA = True
    # BatchNorm (train) fwd / bwd on widths outside the power-of-two family, incl. channel_stats fallback
    for c in (24, 48, 80, 96, 160, 192, 288, 320, 448, 768, 1280):
        m_ = 2 * 9 * 9
        y = cl(bf(torch.randn(2, c, 9, 9, device=dev) * 2 + 0.5))
        g, b = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev) * 0.1
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        yr = y.float().contiguous().requires_grad_(True)
        gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
        zr = torch.relu(F.batch_norm(yr, None, None, gr, br, True, 0.1, 1e-3))
        z, save = nv.bn_act_fwd(y, None, g, b, rm, rv, 1e-3, 0.1, True, None, True)
        report(f"bn fwd C={c}", z, zr, 2e-2)
        dz = cl(bf(torch.randn_like(zr)))
        zr.backward(dz.float().contiguous())
        gg, bg = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        dyv, _, _ = nv.bn_act_bwd(dz, z, y, save, g, True, False, gg, bg, beta=b, had_residual=False)
        report(f"bn bwd dx C={c}", dyv, yr.grad, 3e-2)
        report("   dgamma", gg, gr.grad, 2e-2, atol=2e-2)
        report("   dbeta", bg, br.grad, 2e-2, atol=2e-2)


def g_conv_dgrad():
    import torch

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    cases = [(2, 64, 56, 56, 128, 3, 2, 1), (3, 256, 14, 14, 512, 1, 2, 0), (2, 128, 13, 13, 128, 3, 2, 1), (3, 64, 7, 7, 64, 3, 1, 1), (5, 128, 14, 14, 128, 3, 1, 1), (2, 64, 56, 56, 128, 3, 1, 1), (2, 64, 28, 28, 64, 3, 1, 1), (2, 64, 15, 15, 64, 3, 1, 0), (1, 64, 20, 20, 64, 3, 1, 2), (2, 64, 8, 8, 64, 3, 1, 1), (2, 64, 9, 9, 128, 3, 2, 1), (2, 128, 14, 14, 128, 3, 1, 1),
             (2, 256, 8, 8, 512, 1, 2, 0), (2, 256, 7, 7, 64, 1, 1, 0), (2, 64, 12, 12, 192, 5, 1, 2),
             (2, 128, 28, 28, 128, 3, 2, 1)]
    for (n, ci, h, w_, co, k, s, p) in cases:
        x = torch.randn(n, ci, h, w_, device=dev).float().requires_grad_(True)
        w = bf(torch.randn(co, ci, k, k, device=dev) * (1.0 / (co * k * k) ** 0.5))
        yr = _conv_ref(x, w, s, p)
        dy = cl(bf(torch.randn_like(yr)))
        yr.backward(dy.float())
        dx = nv.conv_dgrad(dy, _w_bf16(w), x.shape, (k, k), s, p)
        report(f"conv_dgrad n{n} c{ci} {h}x{w_} <-{co} k{k}s{s}p{p}", dx, x.grad, 2e-2)
    # epilogue add
    add = cl(bf(torch.randn(2, 64, 8, 8, device=dev)))
    x = torch.randn(2, 64, 8, 8, device=dev).requires_grad_(True)
    w = bf(torch.randn(64, 64, 3, 3, device=dev) * 0.05)
    yr = _conv_ref(x, w, 1, 1)
    dy = cl(bf(torch.randn_like(yr)))
    yr.backward(dy.float())
    dx = nv.conv_dgrad(dy, _w_bf16(w), x.shape, (3, 3), 1, 1, add=add)
    report("conv_dgrad + add", dx, x.grad + add.float(), 2e-2)
    # BN-backward reduction fused into the dgrad epilogue: dbeta / dgamma sums equal the stand-alone reduce kernel's
    for (n, ci, h, co, k, s_, p_) in [(2, 64, 12, 128, 3, 1, 1), (3, 128, 9, 256, 1, 1, 0), (2, 64, 16, 64, 3, 2, 1),
                                      (2, 96, 10, 160, 1, 1, 0), (4, 256, 14, 64, 1, 1, 0)]:
        xs = (n, ci, h, h)
        w_ = bf(torch.randn(co, ci, k, k, device=dev) * (1.0 / (co * k * k) ** 0.5))
        ho = (h + 2 * p_ - k) // s_ + 1
        dyv = cl(bf(torch.randn(n, co, ho, ho, device=dev)))
        ybn = cl(bf(torch.randn(*xs, device=dev) * 1.5 + 0.3))
        gam, bet = torch.rand(ci, device=dev) + 0.5, torch.randn(ci, device=dev) * 0.3
        save = torch.stack([ybn.float().mean((0, 2, 3)), 1.0 / (ybn.float().var((0, 2, 3), unbiased=False) + 1e-5).sqrt()]).contiguous()
        pre = torch.zeros(2, ci, device=dev)
        d_fused = nv.conv_dgrad(dyv, _w_bf16(w_), xs, (k, k), s_, p_, bn_reduce=(ybn, gam, bet, save, pre))
        d_plain = nv.conv_dgrad(dyv, _w_bf16(w_), xs, (k, k), s_, p_)
        report(f"dgrad+bn-reduce c{ci}<-{co} k{k}s{s_}: dx unchanged", d_fused, d_plain, 1e-6)
        zdummy = torch.empty_like(ybn)
        dy_a, _, scr = nv.bn_act_bwd(d_plain, zdummy, ybn, save, gam, True, False, None, None, beta=bet, had_residual=False)
        report("   dgamma", pre[0], scr[0], 2e-3, atol=2e-3)      # scratch layout: [0] = dgamma, [1] = dbeta
        report("   dbeta", pre[1], scr[1], 2e-3, atol=2e-3)
        dy_b, _, _ = nv.bn_act_bwd(d_plain, zdummy, ybn, save, gam, True, False, None, None, beta=bet, had_residual=False,
                                   pre_reduced=pre)
        report("   bn apply from fused sums", dy_b, dy_a, 2e-3)
    # epilogue add gated by a ReLU bit mask (shortcut gradient of an identity residual block)
    zpos = torch.rand(2, 64, 8, 8, device=dev) > 0.5
    bits = cl(zpos.to(torch.uint8)).permute(0, 2, 3, 1).reshape(-1, 8, 8)       # [M, C/8, 8]
    mask = (bits.to(torch.int32) << torch.arange(8, device=dev, dtype=torch.int32)).sum(-1).to(torch.uint8).contiguous()
    dx = nv.conv_dgrad(dy, _w_bf16(w), x.shape, (3, 3), 1, 1, add=add, add_mask=mask)
    report("conv_dgrad + masked add", dx, x.grad + add.float() * zpos.float(), 2e-2)
    x1 = torch.randn(2, 64, 8, 8, device=dev).requires_grad_(True)
    w1 = bf(torch.randn(128, 64, 1, 1, device=dev) * 0.1)
    y1 = _conv_ref(x1, w1, 1, 0)
    dy1 = cl(bf(torch.randn_like(y1)))
    y1.backward(dy1.float())
    dx1 = nv.conv_dgrad(dy1, _w_bf16(w1), x1.shape, (1, 1), 1, 0, add=add, add_mask=mask)
    report("conv_dgrad 1x1 + masked add", dx1, x1.grad + add.float() * zpos.float(), 2e-2)


def g_conv_wgrad():
    import torch

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    cases = [(2, 64, 56, 56, 128, 3, 2, 1), (3, 256, 14, 14, 512, 1, 2, 0), (2, 128, 13, 13, 128, 3, 2, 1), (3, 64, 7, 7, 64, 3, 1, 1), (5, 128, 14, 14, 128, 3, 1, 1), (2, 64, 56, 56, 128, 3, 1, 1), (2, 64, 28, 28, 64, 3, 1, 1), (2, 64, 15, 15, 64, 3, 1, 0), (1, 64, 20, 20, 64, 3, 1, 2), (2, 64, 8, 8, 64, 3, 1, 1), (2, 64, 9, 9, 128, 3, 2, 1), (3, 128, 14, 14, 128, 3, 1, 1),
             (2, 256, 8, 8, 512, 1, 2, 0), (4, 256, 7, 7, 64, 1, 1, 0), (2, 64, 12, 12, 192, 5, 1, 2),
             (8, 64, 56, 56, 64, 3, 1, 1), (8, 512, 7, 7, 2048, 1, 1, 0)]
    for (n, ci, h, w_, co, k, s, p) in cases:
        x = cl(bf(torch.randn(n, ci, h, w_, device=dev)))
        w = torch.randn(co, ci, k, k, device=dev).requires_grad_(True)
        yr = _conv_ref(x, w, s, p)
        dy = cl(bf(torch.randn_like(yr)))
        yr.backward(dy.float())
        gw = cl(torch.zeros(co, ci, k, k, device=dev))
        nv.conv_wgrad(x, dy, gw, (k, k), s, p)
        report(f"conv_wgrad n{n} c{ci} {h}x{w_} ->{co} k{k}s{s}p{p}", gw, w.grad, 2e-2)
    for tma in (True, False):
        nv.USE_STEM_TMA = tma
        for (k, s, p, hw) in [(7, 2, 3, 32), (11, 4, 2, 63), (3, 1, 1, 16), (3, 2, 0, 35), (7, 2, 0, 41), (7, 2, 3, 224)]:
            img = torch.randn(2, 3, hw, hw, device=dev)
            x4 = nv.nchw_to_nhwc4(img)
            w = torch.randn(64, 3, k, k, device=dev).requires_grad_(True)
            yr = _conv_ref(bf(img), w, s, p)
            dy = cl(bf(torch.randn_like(yr)))
            yr.backward(dy.float())
            gw = cl(torch.zeros(64, 3, k, k, device=dev))
            nv.conv_wgrad(x4, dy, gw, (k, k), s, p)
            report(f"stem wgrad {'tma' if tma else 'gather'} k{k}s{s}p{p}", gw, w.grad, 2e-2)
    nv.USE_STEM_TMA = True


def g_linear():
    import torch

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    for (B, K, N) in [(256, 2048, 1000), (64, 512, 1000), (32, 9216, 4096)]:
        x = bf(torch.randn(B, K, device=dev))
        w = torch.randn(N, K, device=dev) * 0.02
        b = torch.randn(N, device=dev)
        y = nv.linear_fwd(x, bf(w), b)
        ref = x.float() @ bf(w).float().t() + b
        report(f"linear fwd B{B} K{K} N{N}", y[:, :N], ref, 2e-2)
        RESULTS.append(y[:, N:].abs().max().item() == 0 if y.shape[1] > N else True)
        dy = torch.zeros_like(y)
        dy[:, :N] = bf(torch.randn(B, N, device=dev))
        dx = nv.linear_dgrad(dy, bf(w))
        report(f"linear dgrad B{B} K{K} N{N}", dx, dy[:, :N].float() @ bf(w).float(), 2e-2)
        gw = torch.zeros(N, K, device=dev)
        nv.linear_wgrad(x, dy, gw)
        report(f"linear wgrad B{B} K{K} N{N}", gw, dy[:, :N].float().t() @ x.float(), 2e-2)


def _unpack_mask(mask, numel):
    """[M, C/8] uint8 bit mask -> float {0,1} vector of M*C elements (bit i of byte [m][c/8] = element [m][c + i])."""
    import torch

    bits = (mask.reshape(-1, 1).to(torch.int32) >> torch.arange(8, device=mask.device, dtype=torch.int32)) & 1
    return bits.reshape(-1)[:numel].float()


def g_bn():
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    dev = "cuda"
    for (n, c, h, relu, res) in [(4, 64, 14, True, False), (2, 256, 7, True, True), (3, 2048, 4, False, False), (2, 128, 9, True, True)]:
        y = cl(bf(torch.randn(n, c, h, h, device=dev) * 2 + 0.5))
        r = cl(bf(torch.randn(n, c, h, h, device=dev))) if res else None
        gamma, beta = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev)
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        z, save = nv.bn_act_fwd(y, None, gamma, beta, rm, rv, 1e-5, 0.1, relu, r, True)
        yr = y.float().requires_grad_(True)
        gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        rm2, rv2 = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        zr = F.batch_norm(yr, rm2, rv2, gr, br, True, 0.1, 1e-5)
        rr = r.float().requires_grad_(True) if res else None
        if res:
            zr = zr + rr
        if relu:
            zr = torch.relu(zr)
        report(f"bn_act fwd c{c} relu={relu} res={res}", z, zr.detach(), 2e-2)
        report("  running_mean", rm, rm2, 1e-3, atol=1e-3)
        report("  running_var", rv, rv2, 1e-2)
        dz = cl(bf(torch.randn_like(zr)))
        zr.backward(dz.float())
        gg, bg = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        dy, dres, _ = nv.bn_act_bwd(dz, z, y, save, gamma, relu, res, gg, bg)
        report("  bwd dy", dy, yr.grad, 3e-2)
        report("  bwd dgamma", gg, gr.grad, 2e-2)
        report("  bwd dbeta", bg, br.grad, 2e-2)
        if res:
            report("  bwd dres", dres, rr.grad, 2e-2)
        if res and relu:
            # 1-bit ReLU mask path (what the residual blocks use): identical results without reading z in backward
            # (the per-channel sums are accumulated with atomics, i.e. in a run-dependent order: two launches may differ
            #  in the last bit of a sum, which can move an output across a bf16 rounding boundary.  The forward pair
            #  therefore shares ONE statistics tensor and must agree exactly; the backward pair may differ by one bf16 ulp)
            st_shared = torch.stack([y.float().sum((0, 2, 3)), (y.float() ** 2).sum((0, 2, 3))]).contiguous()
            z1, save1 = nv.bn_act_fwd(y, st_shared, gamma, beta, torch.zeros(c, device=dev), torch.ones(c, device=dev), 1e-5, 0.1,
                                      relu, r, True)
            rm3, rv3 = torch.zeros(c, device=dev), torch.ones(c, device=dev)
            z2, save2, zmask = nv.bn_act_fwd(y, st_shared, gamma, beta, rm3, rv3, 1e-5, 0.1, relu, r, True, want_mask=True)
            report("  bitmask fwd z", z2, z1, 1e-6)
            report("  bitmask == (z > 0)", _unpack_mask(zmask, z2.numel()), (z2.permute(0, 2, 3, 1).reshape(-1) > 0).float(), 1e-6)
            gg1, bg1 = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
            dy1, dres1, _ = nv.bn_act_bwd(dz, z1, y, save1, gamma, relu, True, gg1, bg1)
            gg2, bg2 = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
            dy2, dres2, _ = nv.bn_act_bwd(dz, None, y, save2, gamma, relu, True, gg2, bg2, zmask=zmask)
            report_abs("  bitmask bwd dy", dy2, dy1, 2.0 ** -7, 1e-6)
            report("  bitmask bwd dres", dres2, dres1, 1e-6)
            report("  bitmask bwd dgamma", gg2, gg1, 1e-5)
    # fused stem: maxpool(relu(BN(y))) forward without the BN output, backward rebuilt from the pooled gradient
    for (n, c, h, w_) in [(2, 64, 16, 16), (3, 96, 11, 13), (2, 64, 112, 112)]:
        y = cl(bf(torch.randn(n, c, h, w_, device=dev) * 2 + 0.5))
        gamma, beta = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev) * 0.5
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        stats = torch.stack([y.float().sum((0, 2, 3)), (y.float() ** 2).sum((0, 2, 3))]).contiguous()
        pooled, arg, save = nv.bn_relu_maxpool_fwd(y, stats, gamma, beta, rm, rv, 1e-5, 0.1, 3, 2, 1)
        yr = y.float().contiguous().requires_grad_(True)
        gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        rm2, rv2 = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        pr = F.max_pool2d(torch.relu(F.batch_norm(yr, rm2, rv2, gr, br, True, 0.1, 1e-5)), 3, 2, 1)
        report(f"stem bn+relu+maxpool fwd c{c} {h}x{w_}", pooled, pr.detach(), 2e-2)
        report("  running_var", rv, rv2, 1e-2)
        dp = cl(bf(torch.randn_like(pr)))
        pr.backward(dp.float().contiguous())
        gg, bg = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        dyv = nv.bn_pool_bwd(dp, arg, y, save, gamma, beta, gg, bg, 3, 2, 1)
        # reference for dy: the unfused native kernels (same bf16 rounding of z, hence the same arg-max on ties; the
        # fp32 torch graph above picks a different pixel wherever two window values round to the same bf16)
        z_u, save_u = nv.bn_act_fwd(y, stats, gamma, beta, torch.zeros(c, device=dev), torch.ones(c, device=dev), 1e-5, 0.1,
                                    True, None, True)
        p_u, arg_u = nv.maxpool_fwd(z_u, 3, 2, 1)
        dz_u = nv.maxpool_bwd(dp, arg_u, z_u.shape, 3, 2, 1)
        dy_u, _, _ = nv.bn_act_bwd(dz_u, z_u, y, save_u, gamma, True, False, None, None, beta=beta, had_residual=False)
        report("  stem fwd == unfused", pooled, p_u, 1e-6)
        report("  stem bwd dy (vs unfused native)", dyv, dy_u, 2e-2)
        report("  stem bwd dgamma", gg, gr.grad, 2e-2, atol=1e-1)
        report("  stem bwd dbeta", bg, br.grad, 2e-2, atol=1e-1)
    # odd widths (chunked thread mapping) with the bit mask
    for c in (96, 320):
        y = cl(bf(torch.randn(2, c, 6, 6, device=dev)))
        r = cl(bf(torch.randn(2, c, 6, 6, device=dev)))
        gamma, beta = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev)
        rm, rv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        st_shared = torch.stack([y.float().sum((0, 2, 3)), (y.float() ** 2).sum((0, 2, 3))]).contiguous()
        z, save = nv.bn_act_fwd(y, st_shared, gamma, beta, rm.clone(), rv.clone(), 1e-5, 0.1, True, r, True)
        z2, save2, zmask = nv.bn_act_fwd(y, st_shared, gamma, beta, rm, rv, 1e-5, 0.1, True, r, True, want_mask=True)
        dz = cl(bf(torch.randn_like(z.float())))
        g1, b1, g2, b2 = (torch.zeros(c, device=dev) for _ in range(4))
        dy, dres, _ = nv.bn_act_bwd(dz, z, y, save, gamma, True, True, g1, b1)
        dy2, dres2, _ = nv.bn_act_bwd(dz, None, y, save2, gamma, True, True, g2, b2, zmask=zmask)
        report_abs(f"  bitmask C={c} dy", dy2, dy, 2.0 ** -7, 1e-6)      # one bf16 ulp: see the atomics note above
        report(f"  bitmask C={c} dres", dres2, dres, 1e-6)


def g_sgd():
    import torch

    from distributeddeeplearning_b200.parallel import dist
    from distributeddeeplearning_b200.parallel.engine import FusedSGD

    dist.init()
    for (mom, wd, nest) in [(0.0, 0.0, False), (0.9, 5e-5, False), (0.9, 1e-4, True)]:
        torch.manual_seed(0)
        ps = [torch.nn.Parameter(torch.randn(s, device="cuda")) for s in [(64, 3, 7, 7), (1000, 512), (77,), (256, 64, 3, 3)]]
        ref = [torch.nn.Parameter(p.detach().clone()) for p in ps]
        opt = FusedSGD(ps, lr=0.1, momentum=mom, weight_decay=wd, nesterov=nest, debug=True)
        ropt = torch.optim.SGD(ref, lr=0.1, momentum=mom, weight_decay=wd, nesterov=nest)
        for it in range(3):
            for p, r in zip(ps, ref):
                g = torch.randn_like(r)
                r.grad = g.clone()
                p.grad.add_(g.view_as(p.grad))
                p._ddl_ready()
            opt.step()
            ropt.step()
        torch.cuda.synchronize()
        for i, (p, r) in enumerate(zip(ps, ref)):
            report(f"fused_sgd mom={mom} wd={wd} nest={nest} p{i}", p.detach(), r.detach(), 1e-5)
            report("   bf16 copy", p._ddl_bf16.float().reshape(-1), r.detach().to(torch.bfloat16).float().reshape(-1), 1e-2)
        RESULTS.append(all(float(p.grad.abs().max()) == 0 for p in ps))
        print("grads cleared:", RESULTS[-1])


def _cos(a, b):
    a, b = a.float().reshape(-1), b.float().reshape(-1)
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def g_model():
    """Whole-model check.  bf16 activations vs an fp32 oracle differ by rounding that grows with depth, so
    gradients are judged by cosine similarity / norm ratio against (a) torchvision fp32 and (b) this repo's own
    PyTorch composite run in bf16 (same rounding points, different kernels)."""
    import os

    import torch
    import torchvision

    from distributeddeeplearning_b200 import models, ops

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for name, bs in [("resnet18", 32), ("resnet50", 32)]:
        torch.manual_seed(0)
        # zero-init of the last BN gamma of every block keeps the random-init net well conditioned, so bf16
        # rounding does not swamp the gradient signal (both nets share the same weights either way)
        m = models.get_model(name, zero_init_residual=True).cuda().train()
        tv = getattr(torchvision.models, name)().cuda().train()
        tv.load_state_dict(m.state_dict())
        m2 = models.get_model(name).cuda().train()
        m2.load_state_dict(m.state_dict())
        x = torch.randn(bs, 3, 224, 224, device="cuda").to(torch.bfloat16).float()
        y = torch.randint(0, 1000, (bs,), device="cuda")
        out = m(x)
        loss = ops.softmax_cross_entropy(out, y, 1000)
        loss.backward()
        ro = tv(x)
        rl = torch.nn.functional.cross_entropy(ro, y)
        rl.backward()
        os.environ["DDL_B200_IMPL"] = "torch"
        co = m2(x)
        cl_ = ops.softmax_cross_entropy(co, y, 1000)
        cl_.backward()
        os.environ["DDL_B200_IMPL"] = "native"
        report(f"{name} loss vs fp32", loss.reshape(1), rl.detach().reshape(1), 3e-2)
        print(f"{name} logits cos vs fp32 {_cos(out, ro):.5f}   vs bf16-composite {_cos(out, co):.5f}")
        RESULTS.append(_cos(out, ro) > 0.98)
        gn, gc = dict(m.named_parameters()), dict(m2.named_parameters())
        worst = (1.0, "")
        lag = (0.0, "")
        for k, p in tv.named_parameters():
            if float(p.grad.norm()) == 0.0:
                continue
            c1 = _cos(gn[k].grad, p.grad)
            c2 = _cos(gc[k].grad, p.grad)
            if c1 < worst[0]:
                worst = (c1, k)
            if c2 - c1 > lag[0]:
                lag = (c2 - c1, k)
            if k in ("conv1.weight", "bn1.weight", "layer1.0.conv1.weight", "layer2.0.downsample.0.weight",
                     "layer3.0.conv2.weight", "layer4.0.conv1.weight", "fc.weight", "fc.bias"):
                ratio = float(gn[k].grad.float().norm() / (p.grad.norm() + 1e-30))
                print(f"   {k:32s} cos(native,fp32)={c1:.4f} cos(composite,fp32)={c2:.4f} norm ratio={ratio:.3f}")
        print(f"{name}: worst cosine(native grad, fp32 grad) = {worst[0]:.4f} at {worst[1]}; "
              f"largest deficit vs the bf16 composite = {lag[0]:.4f} at {lag[1]}")
        RESULTS.append(worst[0] > 0.80 and lag[0] < 0.08)


def g_zoo():
    """One short training run per remaining zoo model through the public benchmark session (fused engine included)."""
    import torch

    from distributeddeeplearning_b200.parallel import dist
    from distributeddeeplearning_b200.workloads.benchmark import BenchmarkSession

    dist.init()
    for name, bs in [("vgg16", 32), ("alexnet", 64), ("resnet101", 16), ("resnet34", 32), ("inception_v3", 16),
                     ("vgg11_bn", 16), ("densenet121", 16), ("squeezenet1_1", 32)]:
        torch.manual_seed(0)
        s = BenchmarkSession(name, bs, True, lr=0.01 if "vgg" not in name and name not in ("alexnet", "squeezenet1_1") else 0.001)
        losses = [float(s.step()) for _ in range(6)]
        torch.cuda.synchronize()
        s.optimizer.check_errors()
        finite = all(l == l and abs(l) < 1e4 for l in losses)
        # AlexNet / VGG-16 sit on the ln(1000) plateau for the first few hundred SGD steps: only require no blow-up there
        down = losses[-1] < losses[0] + (0.02 if name in ("alexnet", "vgg16", "squeezenet1_1") else 0.0)
        print(f"[{'ok' if finite and down else 'FAIL'}] {name:14s} batch {bs}: loss " + " ".join(f"{l:.3f}" for l in losses), flush=True)
        RESULTS.append(finite and down)
        del s
        torch.cuda.empty_cache()


def g_graph():
    """Whole-step CUDA-graph replay, incl. a dropout model (device-side step counter) and a BN/residual model."""
    import torch

    from distributeddeeplearning_b200.parallel import dist
    from distributeddeeplearning_b200.workloads.benchmark import BenchmarkSession

    dist.init()
    for name, bs in [("alexnet", 32), ("resnet18", 16), ("squeezenet1_1", 16)]:
        torch.manual_seed(0)
        s = BenchmarkSession(name, bs, True, lr=0.01 if name == "resnet18" else 0.001)
        ok = s.enable_graph(warmup=2)
        losses = [float(s.step()) for _ in range(5)]
        torch.cuda.synchronize()
        s.optimizer.check_errors()
        finite = all(l == l and abs(l) < 1e4 for l in losses)
        print(f"[{'ok' if ok and finite else 'FAIL'}] graph replay {name:14s}: captured={ok} loss " + " ".join(f"{l:.3f}" for l in losses), flush=True)
        RESULTS.append(ok and finite)
        del s
        torch.cuda.empty_cache()


def g_zoograd():
    """Dropout models (no BN): one eval-mode forward/backward against torchvision fp32 with the same weights."""
    import torch
    import torchvision

    from distributeddeeplearning_b200 import models, ops

    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for name, bs in [("alexnet", 32), ("vgg16", 8)]:
        torch.manual_seed(0)
        m = models.get_model(name).cuda().eval()
        tv = getattr(torchvision.models, name)().cuda().eval()
        tv.load_state_dict(m.state_dict())
        x = torch.randn(bs, 3, 224, 224, device="cuda").to(torch.bfloat16).float()
        y = torch.randint(0, 1000, (bs,), device="cuda")
        out = m(x)
        ops.softmax_cross_entropy(out, y, 1000).backward()
        ro = tv(x)
        torch.nn.functional.cross_entropy(ro, y).backward()
        gn = dict(m.named_parameters())
        worst = (1.0, "")
        for k, p in tv.named_parameters():
            c1 = _cos(gn[k].grad, p.grad)
            if c1 < worst[0]:
                worst = (c1, k)
        lc = _cos(out[:, :1000], ro)
        print(f"{name}: logits cos vs fp32 {lc:.5f}; worst grad cosine {worst[0]:.4f} at {worst[1]}", flush=True)
        RESULTS.append(lc > 0.99 and worst[0] > 0.85)   # bf16 activations, 16 layers, small batch: bias grads are the noisiest
        del m, tv
        torch.cuda.empty_cache()


def g_avgdebug():
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    x = cl(bf(torch.randn(1, 8, 5, 5, device="cuda")))
    xr = x.float().contiguous().requires_grad_(True)
    yr = F.avg_pool2d(xr, 3, 1, 1)
    dy = cl(bf(torch.ones_like(yr)))
    yr.backward(dy.float().contiguous())
    got = nv.avgpool_bwd(dy, x.shape, 3, 1, 1, True)
    print("ref", xr.grad[0, 0])
    print("got", got[0, 0].float())
    report("avgpool bwd tiny", got, xr.grad, 1e-2)


def run_group(name):
    fn = globals()["g_" + name]
    fn()
    import torch

    torch.cuda.synchronize()
    from distributeddeeplearning_b200.ops import native as _nv

    stuck = _nv.conv_timeouts(raise_error=False)
    if stuck is not None:
        print("[FAIL]", stuck, flush=True)
        RESULTS.append(False)
    rejected = _nv._TUNE.get("rejected")
    if rejected:
        print("[FAIL] autotuner rejected dead-locking variants:", rejected, flush=True)
        RESULTS.append(False)
    ok = all(RESULTS)
    print(f"== group {name}: {sum(RESULTS)}/{len(RESULTS)} checks passed ==", flush=True)
    return 0 if ok else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--group", default=None)
    ap.add_argument("--timeout", type=int, default=600)
    ap.add_argument("--groups", default=",".join(GROUPS))
    a = ap.parse_args()
    if a.group:
        return run_group(a.group)
    bad = []
    for g in a.groups.split(","):
        t0 = time.time()
        print(f"######## {g}", flush=True)
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--group", g], timeout=a.timeout)
            rc = r.returncode
        except subprocess.TimeoutExpired:
            rc = 124
            print(f"== group {g}: TIMEOUT after {a.timeout}s ==", flush=True)
        print(f"######## {g} rc={rc} {time.time() - t0:.1f}s", flush=True)
        if rc != 0:
            bad.append(g)
    print("FAILED GROUPS:", bad if bad else "none", flush=True)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
