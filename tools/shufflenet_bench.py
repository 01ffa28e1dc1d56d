#!/usr/bin/env python
"""Forward + backward time of every distinct ShuffleNetV2 unit shape of x0.5, x1.0, x1.5 and x2.0 at 224, for three
versions of the unit on the same bf16 channels-last input and weights:

  node       ops.shuffle_unit: one autograd node (branch BN + concat + shuffle in one kernel pass, (lo, hi) halves
             handed to the next unit, widths that are not multiples of 8 zero-padded inside the node)
  layers     the per-layer composition it replaces: one conv_bn node per conv + BN, torch chunk / cat / shuffle; widths
             that are not multiples of 8 fall to conv_bn's torch composite there
  cudnn      torchvision's InvertedResidual in bf16 channels-last (cuDNN)

plus the bytes each one moves, computed from the shapes (activations read and written once per kernel pass, bf16), and
the training throughput of the four models (forward, backward, no optimizer) against torchvision bf16 channels-last.
CUDA events, L2 flushed before every run, median of --iters runs after a warm-up run; the card's name, power limit and
maximum SM clock are printed with the tables.

    python tools/shufflenet_bench.py [--batch 256] [--iters 20] [--model-steps 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from depthwise_bench import card, timed  # noqa: E402


def _p8(c):
    return (c + 7) // 8 * 8


def unit_bytes(inp, oup, stride, hw, n, padded):
    """Activation bytes of one forward + backward of the unit (bf16), counting each tensor a kernel pass reads or
    writes once.  ``padded``: widths rounded up to 8 (the node); the three copies of the composition (chunk, cat,
    shuffle) are added by :func:`composition_bytes`."""
    p = _p8 if padded else (lambda c: c)
    bf = oup // 2
    ho = hw // stride
    mi, mo = n * hw * hw, n * ho * ho
    cb = p(bf)
    fwd = bwd = 0
    if stride == 2:
        ci = p(inp)
        fwd += mi * ci + mo * ci * 2 + mo * ci * 2 + mo * ci + mo * cb       # dw, BN, 1x1 of branch1
        bwd += mo * cb * 2 + mo * ci + mo * ci * 3 + mo * ci * 2 + mi * ci + mo * ci + mi * ci
        src = mi * ci
    else:
        src = mi * cb
    fwd += src + mi * cb + mi * cb * 3 + mi * cb + mo * cb + mo * cb * 3 + mo * cb + mo * cb   # 1x1, BN, dw, BN, 1x1
    fwd += mo * cb * 2 + mo * 2 * cb                                                             # shuffle
    bwd += mo * 2 * cb * 2 + mo * cb * 3 + mo * cb * 2                                           # shuffle backward
    bwd += mo * cb * 2 + mo * cb * 2 + mo * cb * 5 + mo * cb + mi * cb * 2 + mi * cb * 5 + mi * cb + src * 2
    return 2 * (fwd + bwd)


def composition_bytes(inp, oup, stride, hw, n):
    ho = hw // stride
    mo = n * ho * ho
    extra = (n * hw * hw * inp * 2) if stride == 1 else 0       # chunk copy (read + write)
    extra += mo * oup * 2 * 2                                    # cat, shuffle
    return unit_bytes(inp, oup, stride, hw, n, False) + 2 * 2 * extra      # forward and backward copies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--model-steps", type=int, default=20)
    a = ap.parse_args()
    import torch
    import torchvision
    from torchvision.models.shufflenetv2 import InvertedResidual as TvUnit

    from distributeddeeplearning_b200 import models, ops
    from distributeddeeplearning_b200.models.layers import conv_bn
    from distributeddeeplearning_b200.models.shufflenetv2 import InvertedResidual
    from distributeddeeplearning_b200.ops.shufflenet import channel_shuffle
    from gpu_diag import shufflenet_unit_shapes

    if not torch.cuda.is_available():
        raise SystemExit("shufflenet_bench.py needs a GPU")
    dev = torch.device("cuda")
    CL = torch.channels_last
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    info = card()
    n = a.batch
    print(f"# {info} (name, power.limit, clocks.max.sm); batch {n}; unit forward + backward, median of {a.iters} (ms); "
          "GB from shapes")
    print(f"{'unit':>22} | {'node':>7} {'layers':>7} {'cudnn':>7} | {'GB node':>7} {'GB lay':>7} | {'layers/node':>11} "
          f"{'cudnn/node':>10}")
    torch.manual_seed(0)
    rows, seen = [], set()
    for name, inp, oup, stride, hw in shufflenet_unit_shapes():
        if (inp, oup, stride, hw) in seen:
            continue
        seen.add((inp, oup, stride, hw))
        u = InvertedResidual(inp, oup, stride).to(dev).train()
        tv = TvUnit(inp, oup, stride)
        tv.load_state_dict(u.state_dict())
        tv = tv.to(device=dev, dtype=torch.bfloat16, memory_format=CL).train()
        bf = oup // 2
        x = torch.randn(n, inp, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=CL)
        xp = torch.zeros(n, _p8(inp), hw, hw, device=dev, dtype=torch.bfloat16).contiguous(memory_format=CL)
        xp[:, :inp] = x
        if stride == 1:
            lo = torch.zeros(n, _p8(bf), hw, hw, device=dev, dtype=torch.bfloat16).contiguous(memory_format=CL)
            hi = lo.clone()
            lo[:, :bf], hi[:, :bf] = x[:, :bf], x[:, bf:]
        ho = hw // stride
        dzp = torch.randn(n, _p8(bf), ho, ho, device=dev).to(torch.bfloat16).contiguous(memory_format=CL)
        dz = torch.randn(n, oup, ho, ho, device=dev).to(torch.bfloat16).contiguous(memory_format=CL)

        def node():
            if stride == 1:
                li, hi_ = lo.detach().requires_grad_(True), hi.detach().requires_grad_(True)
                torch.autograd.backward(u((li, hi_)), (dzp, dzp))
            else:
                xi = xp.detach().requires_grad_(True)
                torch.autograd.backward(u(xi), (dzp, dzp))

        def layers():
            xi = x.detach().requires_grad_(True)
            b2 = u.branch2
            if stride == 1:
                x1, x2 = xi.chunk(2, dim=1)
                x2 = x2.contiguous(memory_format=CL)
            else:
                b1 = u.branch1
                x1 = conv_bn(conv_bn(xi, b1[0], b1[1], relu=False), b1[2], b1[3])
                x2 = xi
            h = conv_bn(x2, b2[0], b2[1])
            h = conv_bn(h, b2[3], b2[4], relu=False)
            h = conv_bn(h, b2[5], b2[6])
            out = channel_shuffle(torch.cat((x1, h), 1), 2).contiguous(memory_format=CL)
            out.backward(dz)

        def cudnn():
            xi = x.detach().requires_grad_(True)
            tv(xi).backward(dz)

        t = [timed(f, a.iters, flush) / 1e3 for f in (node, layers, cudnn)]
        gb = (unit_bytes(inp, oup, stride, hw, n, True) / 1e9, composition_bytes(inp, oup, stride, hw, n) / 1e9)
        r = {"unit": f"{inp}->{oup} s{stride} {hw}", "models": name, "node_ms": t[0], "layers_ms": t[1],
             "cudnn_ms": t[2], "node_GB": gb[0], "layers_GB": gb[1]}
        rows.append(r)
        print(f"{r['unit']:>22} | {t[0]:7.3f} {t[1]:7.3f} {t[2]:7.3f} | {gb[0]:7.3f} {gb[1]:7.3f} | "
              f"{t[1] / t[0]:11.3f} {t[2] / t[0]:10.3f}", flush=True)
        del u, tv
        torch.cuda.empty_cache()
    print(f"# training throughput (forward + backward + loss, no optimizer), batch {n}, img/s")
    thr = []
    for name in ("shufflenet_v2_x0_5", "shufflenet_v2_x1_0", "shufflenet_v2_x1_5", "shufflenet_v2_x2_0"):
        m = models.get_model(name).to(dev).train()
        tv = getattr(torchvision.models, name)().to(device=dev, dtype=torch.bfloat16, memory_format=CL).train()
        x = torch.randn(n, 3, 224, 224, device=dev)
        xb = x.to(torch.bfloat16).contiguous(memory_format=CL)
        y = torch.randint(0, 1000, (n,), device=dev)

        def ours():
            ops.softmax_cross_entropy(m(x), y, 1000).backward()

        def theirs():
            torch.nn.functional.cross_entropy(tv(xb).float(), y).backward()

        res = {}
        for label, f in (("ours", ours), ("torchvision", theirs)):
            for _ in range(3):
                f()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.model_steps):
                f()
            e1.record()
            e1.synchronize()
            res[label] = n * a.model_steps / (e0.elapsed_time(e1) / 1e3)
        thr.append({"model": name, **res})
        print(f"{name:>20}: ours {res['ours']:9.0f}  torchvision bf16 channels-last {res['torchvision']:9.0f}  "
              f"ratio {res['ours'] / res['torchvision']:.3f}", flush=True)
        del m, tv
        torch.cuda.empty_cache()
    print("JSON " + json.dumps({"device": info, "batch": n, "rows": rows, "throughput": thr}))


if __name__ == "__main__":
    sys.exit(main())
