#!/usr/bin/env python
"""Forward + backward time of every residual Fused-MBConv shape of EfficientNetV2-S, -M and -L at its input size, for
three versions of the block on the same bf16 channels-last input, weights and stochastic-depth vector:

  node       ops.fused_mbconv: one autograd node (BN code 6, or the projection BN's stochastic depth; the residual's
             gradient added in the 3x3 data gradient's store)
  layers     the per-layer composition the node replaces: one conv_bn node per layer; without an expansion the scale and
             the residual add are separate elementwise ops and autograd sums the two gradients of x
  cudnn      torch.nn Conv2d / BatchNorm2d / SiLU modules in bf16 channels-last (cuDNN), the scale and add in torch

CUDA events, L2 flushed before every run, median of --iters runs after a warm-up run; the card's name, power limit and
maximum SM clock are printed with the table.

    python tools/efficientnet_v2_bench.py [--batch 128] [--iters 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from depthwise_bench import card, timed  # noqa: E402

# residual Fused-MBConv blocks as (C, expand, H=W) -> the models (at their input size) that have them
SHAPES = {(24, 1, 192): "S", (48, 4, 96): "S", (64, 4, 48): "S", (24, 1, 240): "M", (48, 4, 120): "M",
          (80, 4, 60): "M", (32, 1, 240): "L", (64, 4, 120): "L", (96, 4, 60): "L"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    import torch.nn as nn

    from distributeddeeplearning_b200 import ops
    from distributeddeeplearning_b200.models.efficientnet_v2 import _BN, FusedMBConv
    from distributeddeeplearning_b200.ops.efficientnet_v2 import fused_mbconv_layers

    if not torch.cuda.is_available():
        raise SystemExit("efficientnet_v2_bench.py needs a GPU")
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    info = card()
    print(f"# {info} (name, power.limit, clocks.max.sm); batch {a.batch}; forward + backward, median of {a.iters} (ms)")
    print(f"{'C':>3} {'e':>1} {'HW':>3} {'model':>5} | {'node':>7} {'layers':>7} {'cudnn':>7} | {'layers/node':>11}")
    torch.manual_seed(0)
    keep = ops.stochastic_depth_keep(a.batch, 0.1, dev)
    rows = []
    for (c, e, hw), model in SHAPES.items():
        blk = FusedMBConv(e, 3, 1, c, c, 0.1, _BN).to(dev).train()
        mods = [m for layer in blk.block for m in (layer[0], layer[1])]
        ref = nn.Sequential()
        for i, layer in enumerate(blk.block):
            conv = nn.Conv2d(layer[0].in_channels, layer[0].out_channels, layer[0].kernel_size, 1, layer[0].padding,
                             bias=False)
            ref.append(conv)
            ref.append(nn.BatchNorm2d(layer[0].out_channels, eps=1e-3))
            if i == 0:
                ref.append(nn.SiLU())
        ref = ref.to(device=dev, dtype=torch.bfloat16, memory_format=torch.channels_last).train()
        x = torch.randn(a.batch, c, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dz = torch.randn_like(x)
        kh = keep.to(torch.bfloat16).view(-1, 1, 1, 1)

        def run(f):
            def step():
                xi = x.detach().requires_grad_(True)
                f(xi).backward(dz)
            return step

        node = run(lambda xi: ops.fused_mbconv(xi, *mods, keep=keep))
        layers = run(lambda xi: fused_mbconv_layers(xi, *mods, keep=keep))
        cudnn = run(lambda xi: ref(xi) * kh + xi)
        xi = x.detach().requires_grad_(True)
        assert type(ops.fused_mbconv(xi, *mods, keep=keep).grad_fn).__name__ == "_FusedMBConvBackward"
        t = [timed(f, a.iters, flush) / 1e3 for f in (node, layers, cudnn)]
        r = {"C": c, "expand": e, "HW": hw, "model": model, "node_ms": t[0], "layers_ms": t[1], "cudnn_ms": t[2]}
        rows.append(r)
        print(f"{c:3d} {e:1d} {hw:3d} {model:>5} | {t[0]:7.3f} {t[1]:7.3f} {t[2]:7.3f} | {t[1] / t[0]:11.3f}", flush=True)
        del blk, ref, x, dz
        torch.cuda.empty_cache()
    print("JSON " + json.dumps({"device": info, "batch": a.batch, "rows": rows}))


if __name__ == "__main__":
    sys.exit(main())
