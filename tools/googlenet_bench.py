#!/usr/bin/env python
"""Forward + backward time of GoogLeNet's nine Inception module shapes at 224, for three versions of the module on the
same bf16 channels-last input and weights:

  node       ops.inception_module: one autograd node (the three 1x1 convolutions on x as one GEMM, segmented BN + ReLU
             writing the output slices in place, one store of dx)
  layers     the per-layer composition Inception-v3 uses: one conv_bn node per conv + BN, max_pool2d, concat_channels
  cudnn      torchvision's Inception in bf16 channels-last (cuDNN)

plus the bytes each one moves, computed from the shapes (activations read and written once per kernel pass, bf16), and
the training throughput of googlenet and mnasnet1_0 (forward, backward, no optimizer) against torchvision bf16
channels-last.  CUDA events, L2 flushed before every run, median of --iters runs after a warm-up run; the card's name,
power limit and maximum SM clock are printed with the tables.

    python tools/googlenet_bench.py [--batch 256] [--iters 20] [--model-steps 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from depthwise_bench import card, timed  # noqa: E402


def module_bytes(shape, n, node):
    """Activation bytes of one forward + backward of the module (bf16), each tensor a kernel pass reads or writes
    counted once.  The composition reads x three more times (three 1x1 GEMMs and their data gradients read / write
    separately), writes the concat and split copies and sums four input gradients."""
    cin, c1, c2r, c2, c3r, c3, c4, hw = shape
    m = n * hw * hw
    cr, cout = c1 + c2r + c3r, c1 + c2 + c3 + c4
    fwd = m * cin * 2 + m * cin                                  # max-pool: read x, write p (+ arg-max codes)
    fwd += m * cin + m * cr                                      # 1x1 GEMM(s)
    fwd += m * cr * 2                                            # BN1 / BN2r / BN3r
    fwd += m * (c2r + c2 + c3r + c3) + m * (cin + c4)            # 3x3 convs, pool projection
    fwd += m * (c2 + c3 + c4) * 2                                # BN2 / BN3 / BN4
    bwd = m * cout * 2 + m * (c1 + c2 + c3 + c4) * 3             # BN backward: dz, x (reduce), dz, x, dx (apply)
    bwd += m * (c2 + c3) + m * (c2r + c3r) * 5 + m * c4 + m * cin  # 3x3 / pool-projection dgrad, BN2r / BN3r backward
    bwd += m * cin * 2                                           # max-pool backward
    bwd += m * cr + m * cin * 2                                  # 1x1 dgrad + the pool gradient added in its store
    bwd += m * (cin + cr) + m * (c2r + c2) + m * (c3r + c3) + m * (cin + c4)       # weight gradients
    total = fwd + bwd
    if not node:
        total += m * cin * 2 * 2                                 # two more 1x1 GEMMs and data gradients read x / dR
        total += m * cout * 2 * 2                                # concat forward, split backward
        total += m * cin * 3 * 3                                 # autograd sums four input gradients
    return 2 * total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--model-steps", type=int, default=20)
    a = ap.parse_args()
    import torch
    import torchvision
    from torchvision.models.googlenet import Inception as TvInception

    from distributeddeeplearning_b200 import models, ops
    from distributeddeeplearning_b200.models.googlenet import Inception
    from distributeddeeplearning_b200.models.layers import conv_bn
    from gpu_diag import GOOGLENET_MODULES

    if not torch.cuda.is_available():
        raise SystemExit("googlenet_bench.py needs a GPU")
    dev = torch.device("cuda")
    CL = torch.channels_last
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    info = card()
    n = a.batch
    print(f"# {info} (name, power.limit, clocks.max.sm); batch {n}; module forward + backward, median of {a.iters} (ms); "
          "GB from shapes")
    print(f"{'module':>26} | {'node':>7} {'layers':>7} {'cudnn':>7} | {'GB node':>7} {'GB lay':>7} | {'layers/node':>11} "
          f"{'cudnn/node':>10}")
    torch.manual_seed(0)
    rows = []
    for shape in GOOGLENET_MODULES:
        cin, c1, c2r, c2, c3r, c3, c4, hw = shape
        u = Inception(cin, c1, c2r, c2, c3r, c3, c4).to(dev).train()
        tv = TvInception(cin, c1, c2r, c2, c3r, c3, c4)
        tv.load_state_dict(u.state_dict())
        tv = tv.to(device=dev, dtype=torch.bfloat16, memory_format=CL).train()
        x = torch.randn(n, cin, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=CL)
        dz = torch.randn(n, c1 + c2 + c3 + c4, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=CL)

        def node():
            xi = x.detach().requires_grad_(True)
            u(xi).backward(dz)

        def layers():
            xi = x.detach().requires_grad_(True)
            b1 = conv_bn(xi, u.branch1.conv, u.branch1.bn)
            b2 = conv_bn(conv_bn(xi, u.branch2[0].conv, u.branch2[0].bn), u.branch2[1].conv, u.branch2[1].bn)
            b3 = conv_bn(conv_bn(xi, u.branch3[0].conv, u.branch3[0].bn), u.branch3[1].conv, u.branch3[1].bn)
            b4 = conv_bn(ops.max_pool2d(xi, 3, 1, 1, ceil_mode=True), u.branch4[1].conv, u.branch4[1].bn)
            ops.concat_channels([b1, b2, b3, b4]).backward(dz)

        def cudnn():
            xi = x.detach().requires_grad_(True)
            tv(xi).backward(dz)

        t = [timed(f, a.iters, flush) / 1e3 for f in (node, layers, cudnn)]
        gb = (module_bytes(shape, n, True) / 1e9, module_bytes(shape, n, False) / 1e9)
        r = {"module": f"{cin}->{c1}/{c2r}-{c2}/{c3r}-{c3}/{c4} {hw}", "node_ms": t[0], "layers_ms": t[1],
             "cudnn_ms": t[2], "node_GB": gb[0], "layers_GB": gb[1]}
        rows.append(r)
        print(f"{r['module']:>26} | {t[0]:7.3f} {t[1]:7.3f} {t[2]:7.3f} | {gb[0]:7.3f} {gb[1]:7.3f} | "
              f"{t[1] / t[0]:11.3f} {t[2] / t[0]:10.3f}", flush=True)
        del u, tv
        torch.cuda.empty_cache()
    tn, tl = sum(r["node_ms"] for r in rows), sum(r["layers_ms"] for r in rows)
    slower = [r["module"] for r in rows if r["node_ms"] > r["layers_ms"]]
    print(f"# nine modules: node {tn:.3f} ms, layers {tl:.3f} ms (layers/node {tl / tn:.3f}); node slower on: "
          f"{slower or 'none'}")
    print(f"# training throughput (forward + backward + loss, no optimizer), batch {n}, img/s")
    thr = []
    for name in ("googlenet", "mnasnet1_0"):
        m = models.get_model(name).to(dev).train()
        kw = {"init_weights": True} if name == "googlenet" else {}
        tv = getattr(torchvision.models, name)(**kw).to(device=dev, dtype=torch.bfloat16, memory_format=CL).train()
        x = torch.randn(n, 3, 224, 224, device=dev)
        xb = x.to(torch.bfloat16).contiguous(memory_format=CL)
        y = torch.randint(0, 1000, (n,), device=dev)
        w = getattr(m, "aux_loss_weight", None)

        def ours():
            ops.aux_classification_loss(m(x), y, 1000, w).backward()

        def theirs():
            o = tv(xb)
            if isinstance(o, tuple):
                loss = torch.nn.functional.cross_entropy(o[0].float(), y) + w * sum(
                    torch.nn.functional.cross_entropy(t.float(), y) for t in o[1:])
            else:
                loss = torch.nn.functional.cross_entropy(o.float(), y)
            loss.backward()

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
    print("JSON " + json.dumps({"device": info, "batch": n, "rows": rows, "node_ms_total": tn, "layers_ms_total": tl,
                               "node_slower": slower, "throughput": thr}))


if __name__ == "__main__":
    sys.exit(main())
