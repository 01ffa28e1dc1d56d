#!/usr/bin/env python
"""Where does the forward epilogue's time go?  Times the store-bound ResNet-50 layers with epilogue phases switched off
(variant-word bits 12-14, see conv_gemm.cu kDbg*): the outputs are then wrong, only the TIMES mean something.
Also prints the plain write / copy bandwidth of an output-sized buffer for orientation."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributeddeeplearning_b200.ops import native as nv  # noqa: E402
from layer_bench import timeit  # noqa: E402

dev = torch.device("cuda")
cl = torch.channels_last
B = 256
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
SHAPES = [(64, 56, 256, 1, 1, 0), (128, 28, 512, 1, 1, 0), (256, 14, 1024, 1, 1, 0), (64, 56, 64, 3, 1, 1),
          (256, 56, 64, 1, 1, 0)]
DBG = [(0, "full"), (1, "-stats"), (2, "-store"), (3, "-stats-store"), (4, "-drain"), (7, "nothing")]
for (ci, hw, co, k, s, p) in SHAPES:
    x = torch.randn(B, ci, hw, hw, device=dev, dtype=torch.bfloat16).contiguous(memory_format=cl)
    w = torch.randn(co, ci, k, k, device=dev) * 0.05
    wb = w.permute(0, 2, 3, 1).reshape(co, -1).contiguous().to(torch.bfloat16)
    y, _ = nv.conv_fwd(x, wb, (k, k), s, p, stats=True, cout=co)
    y2 = torch.empty_like(y)
    t_set = timeit(lambda: y2.zero_(), reps=3, flush=flush) * 1e3
    t_cpy = timeit(lambda: y2.copy_(y), reps=3, flush=flush) * 1e3
    mb = y.numel() * 2 / 1e6
    print(f"== {ci}x{hw}->{co} k{k}: out {mb:.0f} MB, in {x.numel() * 2 / 1e6:.0f} MB; memset {t_set:.1f} us "
          f"({mb / t_set * 1e3:.0f} GB/s), copy {t_cpy:.1f} us ({2 * mb / t_cpy * 1e3:.0f} GB/s r+w)", flush=True)
    for base, name in ((2, "persistent"), (1, "one-tile"), (2 | (1 << 8), "persistent-pair")):
        row = []
        for d, dn in DBG:
            nv.force_variant(base | (d << 12))
            try:
                t = timeit(lambda: nv.conv_fwd(x, wb, (k, k), s, p, stats=True, cout=co), reps=3, flush=flush) * 1e3
                row.append(f"{dn} {t:.1f}")
            except RuntimeError as e:
                row.append(f"{dn} n/a")
                break
        nv.force_variant(None)
        print(f"   {name:12s}: " + " | ".join(row), flush=True)
    for st in (False,):
        nv.force_variant(2)
        t = timeit(lambda: nv.conv_fwd(x, wb, (k, k), s, p, stats=st, cout=co), reps=3, flush=flush) * 1e3
        nv.force_variant(None)
        print(f"   persistent, stats=False kernel: {t:.1f} us")
