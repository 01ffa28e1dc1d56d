#!/usr/bin/env python
"""Per-stage timing of the ConvNeXt row kernels at batch 256: LayerNorm over channels (forward, backward with the dgamma /
dbeta reduction), exact GELU on fc1's 4C-wide output (forward, backward with fc1's bias reduction) and layer scale +
stochastic depth + residual (forward, backward with the layer-scale and fc2 bias reductions), against PyTorch on the
same bf16 channels-last tensors: aten.native_layer_norm / native_layer_norm_backward, F.gelu / aten.gelu_backward plus
the column sum, and the torch composite of the layer scale.  CUDA events, L2 flushed before every run, median of --iters
runs.

The kernels are bound by HBM bandwidth, so each row also gives the achieved bandwidth from the bytes the pass must move
(LayerNorm forward: read x, write y; backward: read x and dy, write dx; GELU forward: read h, write g; backward: read dg
and h, write dh; layer scale forward: read y and x, write z; backward: read dz and y, write dy) and its fraction of the
H100 SXM data sheet's 3.35 TB/s.  The card's name, power limit and maximum SM clock are printed with the table.  The
widths of ConvNeXt-Base (128..1024) and -Large (192..1536) cover the LayerNorm instantiations that run one block per SM.

    python tools/convnext_bench.py [--model convnext_tiny|convnext_base|convnext_large] [--batch 256] [--iters 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from depthwise_bench import HBM_BYTES_PER_S, card, timed  # noqa: E402

WIDTHS = {"convnext_tiny": (96, 192, 384, 768), "convnext_base": (128, 256, 512, 1024),
          "convnext_large": (192, 384, 768, 1536)}
SIZES = (56, 28, 14, 7)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="convnext_tiny", choices=sorted(WIDTHS))
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F

    from distributeddeeplearning_b200.ops import native as nv

    if not torch.cuda.is_available():
        raise SystemExit("convnext_bench.py needs a GPU")
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    info = card()
    print(f"# {info} (name, power.limit, clocks.max.sm); {a.model}, batch {a.batch}, median of {a.iters} (us); GB/s "
          f"from the bytes each pass must move; % of {HBM_BYTES_PER_S / 1e12:.2f} TB/s (bandwidth-bound)")
    print(f"{'op':>14} {'C':>5} {'HW':>3} | {'native':>8} {'torch':>8} {'GB/s':>5} {'%':>3}")
    rows = []

    def act(c, hw):
        return torch.randn(a.batch, c, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

    def rows_of(t):
        return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])          # a view: channels-last memory is [M][C]

    def add(op, c, hw, nbytes, native, ref):
        t_n, t_r = timed(native, a.iters, flush), timed(ref, a.iters, flush)
        gbs = nbytes / (t_n * 1e-6) / 1e9
        r = {"op": op, "C": c, "HW": hw, "bytes": nbytes, "native_us": t_n, "torch_us": t_r, "GBps": gbs,
             "frac_peak": gbs * 1e9 / HBM_BYTES_PER_S}
        rows.append(r)
        print(f"{op:>14} {c:5d} {hw:3d} | {t_n:8.1f} {t_r:8.1f} {gbs:5.0f} {100 * r['frac_peak']:3.0f}", flush=True)

    for c, hw in zip(WIDTHS[a.model], SIZES):
        x, dy = act(c, hw), act(c, hw)
        g, b = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev)
        gg, gb = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        nb = x.numel() * 2
        xr, dyr, gh, bh = rows_of(x), rows_of(dy), g.to(torch.bfloat16), b.to(torch.bfloat16)
        _, mean, rstd = nv.layer_norm_fwd(x, g, b, 1e-6)
        _, tmean, trstd = torch.ops.aten.native_layer_norm(xr, [c], gh, bh, 1e-6)
        add("LN fwd", c, hw, 2 * nb, lambda: nv.layer_norm_fwd(x, g, b, 1e-6),
            lambda: torch.ops.aten.native_layer_norm(xr, [c], gh, bh, 1e-6))
        add("LN bwd", c, hw, 3 * nb, lambda: nv.layer_norm_bwd(dy, x, mean, rstd, g, gg, gb),
            lambda: torch.ops.aten.native_layer_norm_backward(dyr, xr, [c], tmean, trstd, gh, bh, [True, True, True]))
        h, dg = act(4 * c, hw), act(4 * c, hw)
        db = torch.zeros(4 * c, device=dev)
        nh = h.numel() * 2
        add("GELU fwd", 4 * c, hw, 2 * nh, lambda: nv.gelu_fwd(h), lambda: F.gelu(h))
        add("GELU bwd", 4 * c, hw, 3 * nh, lambda: nv.gelu_bwd(dg, h, db),
            lambda: rows_of(torch.ops.aten.gelu_backward(dg, h)).sum(0, dtype=torch.float32))
        y, dz = act(c, hw), act(c, hw)
        ls = torch.rand(c, device=dev)
        keep = (torch.rand(a.batch, device=dev) > 0.1).float() / 0.9
        lsh, kh = ls.to(torch.bfloat16).view(-1, 1, 1), keep.to(torch.bfloat16).view(-1, 1, 1, 1)
        gl, gbias = torch.zeros(c, device=dev), torch.zeros(c, device=dev)

        def ls_bwd_torch():
            d = dz * lsh * kh
            return d, rows_of(dz * kh * y).sum(0, dtype=torch.float32), rows_of(d).sum(0, dtype=torch.float32)

        add("scale fwd", c, hw, 3 * nb, lambda: nv.layer_scale_fwd(y, ls, keep, x), lambda: y * lsh * kh + x)
        add("scale bwd", c, hw, 3 * nb, lambda: nv.layer_scale_bwd(dz, y, ls, keep, gl, gbias), ls_bwd_torch)
        del x, dy, h, dg, y, dz
    tot = {k: sum(r[k] for r in rows) for k in ("native_us", "torch_us")}
    print(f"all rows (us): native={tot['native_us']:.0f} torch={tot['torch_us']:.0f}")
    print("JSON " + json.dumps({"device": info, "model": a.model, "batch": a.batch, "rows": rows, "totals_us": tot}))


if __name__ == "__main__":
    sys.exit(main())
