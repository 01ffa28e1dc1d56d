"""The float64 weight-gradient reference of tools/gpu_diag.py (the yardstick of its `wgrad` GPU group) on the CPU:
``_wgrad_ref64`` against torch.nn.grad.conv2d_weight in float64 over strides, paddings, rectangular kernels, dilation,
groups and batch chunking; its sum of squared products against brute force; the launch geometry the group records;
and that the group's bound does see one missing 64-row K-block at ResNet-50 layer-1 scale."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def diag():
    spec = importlib.util.spec_from_file_location("gpu_diag", os.path.join(ROOT, "tools", "gpu_diag.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _operands(n, cin, h, w, cout, kernel, stride, pad, dil, seed=0):
    """bf16-valued float64 x and dy (what the kernels multiply), dy of the convolution's output shape."""
    g = torch.Generator().manual_seed(seed)
    P = (h + 2 * pad[0] - dil * (kernel[0] - 1) - 1) // stride + 1
    Q = (w + 2 * pad[1] - dil * (kernel[1] - 1) - 1) // stride + 1
    x = torch.randn(n, cin, h, w, generator=g).bfloat16().double()
    dy = torch.randn(n, cout, P, Q, generator=g).bfloat16().double()
    return x, dy


# n, cin, h, w, cout, (R, S), stride, (pad_h, pad_w), dilation, groups
CASES = [
    (2, 8, 9, 9, 6, (3, 3), 1, (1, 1), 1, 1),
    (3, 8, 11, 10, 4, (3, 3), 2, (1, 1), 1, 1),
    (2, 6, 13, 11, 5, (3, 3), 3, (2, 0), 1, 1),
    (2, 8, 10, 13, 8, (1, 7), 1, (0, 3), 1, 1),
    (2, 8, 13, 10, 8, (7, 1), 1, (3, 0), 1, 1),
    (2, 8, 12, 11, 8, (5, 3), 2, (1, 2), 1, 1),
    (2, 8, 10, 10, 8, (3, 3), 1, (2, 2), 2, 1),
    (2, 4, 9, 9, 8, (3, 3), 2, (2, 1), 2, 1),
    (2, 16, 8, 8, 16, (3, 3), 1, (1, 1), 1, 4),
    (2, 16, 9, 7, 32, (3, 3), 2, (1, 0), 1, 4),
    (2, 64, 7, 7, 64, (3, 3), 2, (1, 1), 1, 32),
    (3, 4, 6, 6, 4, (1, 1), 1, (0, 0), 1, 1),
    (2, 8, 1, 1, 8, (3, 3), 1, (1, 1), 1, 1),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"n{c[0]}c{c[1]}-{c[2]}x{c[3]}->{c[4]}-k{c[5][0]}x{c[5][1]}"
                                                      f"s{c[6]}p{c[7][0]},{c[7][1]}d{c[8]}g{c[9]}")
def test_ref64_matches_conv2d_weight(diag, case):
    n, cin, h, w, cout, kernel, stride, pad, dil, groups = case
    x, dy = _operands(n, cin, h, w, cout, kernel, stride, pad, dil)
    got = diag._wgrad_ref64(x, dy, kernel, stride, pad, dil, groups)
    ref = torch.nn.grad.conv2d_weight(x, (cout, cin // groups) + tuple(kernel), dy, stride, pad, dil, groups)
    ref = ref.permute(0, 2, 3, 1)                               # [Cout, Cin / groups, R, S] -> KRSC
    assert got.dtype == torch.float64 and got.shape == ref.shape
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12 * ref.abs().max().item())


def test_ref64_batch_chunks_split_unevenly(diag):
    """7 images in chunks of 3 (3 + 3 + 1) give the one-chunk result; a channels_last bf16 input gives the same."""
    x, dy = _operands(7, 16, 9, 9, 8, (3, 3), 2, (1, 1), 1, seed=1)
    whole = diag._wgrad_ref64(x, dy, (3, 3), 2, 1)
    chunked = diag._wgrad_ref64(x, dy, (3, 3), 2, 1, chunk=3)
    torch.testing.assert_close(chunked, whole, rtol=1e-13, atol=1e-13 * whole.abs().max().item())
    xb = x.bfloat16().contiguous(memory_format=torch.channels_last)
    dyb = dy.bfloat16().contiguous(memory_format=torch.channels_last)
    torch.testing.assert_close(diag._wgrad_ref64(xb, dyb, (3, 3), 2, 1, chunk=2), whole, rtol=1e-13,
                               atol=1e-13 * whole.abs().max().item())


@pytest.mark.parametrize("groups", [1, 2])
def test_sum_of_squares_matches_brute_force(diag, groups):
    """S2[co][r][s][c] = sum over images and output pixels of (dy * x_tap)^2, from the unfolded input."""
    n, cin, h, cout, k, stride, pad = 2, 4, 6, 6, (3, 3), 2, (1, 1)
    x, dy = _operands(n, cin, h, h, cout, k, stride, pad, 1, seed=2)
    s2 = diag._wgrad_ref64(x, dy, k, stride, pad, 1, groups, squares=True)
    cols = F.unfold(x, k, 1, pad, stride).view(n, cin, k[0] * k[1], -1)          # [n, c, r*s, pixels]
    d = dy.reshape(n, cout, -1)
    cg, og = cin // groups, cout // groups
    brute = torch.zeros(cout, k[0] * k[1], cg, dtype=torch.float64)
    for co in range(cout):
        g = co // og
        for c in range(cg):
            prod = d[:, co, None, :] * cols[:, g * cg + c]                         # [n, r*s, pixels]
            brute[co, :, c] = (prod * prod).sum((0, 2))
    torch.testing.assert_close(s2, brute.view(cout, k[0], k[1], cg), rtol=1e-13, atol=0.0)
    assert (s2[:, 0, 0] == 0).sum() == 0          # stride 2 from row / column -1: every tap sees real pixels here
    x1, dy1 = _operands(2, 4, 1, 1, 4, k, 1, pad, 1, seed=3)
    s2 = diag._wgrad_ref64(x1, dy1, k, 1, pad, squares=True)
    assert (s2[:, 1, 1] > 0).all() and int((s2 == 0).sum()) == 4 * 8 * 4      # 1x1 map: 8 of 9 taps are padding


def test_launch_geometry(diag):
    """launch_conv_wgrad's split arithmetic as the group records it, and the one-K-block-last split picker."""
    assert diag._wgrad_geometry(196, 16) == (16, 13, 1, 4)
    assert diag._wgrad_geometry(196, 16, force_stages=3) == (16, 13, 1, 3)
    assert diag._wgrad_geometry(196, 16, force_stages=3, tma_fed=False) == (16, 13, 1, 4)
    assert diag._wgrad_geometry(4, 3) == (2, 2, 2, 2)
    assert diag._wgrad_geometry(5, 1, force_stages=1) == (1, 5, 5, 2)    # a wrapping ring needs 2 stages
    for total_kb in range(1, 700):
        for req in (1, 2, 3, 7, total_kb - 1, total_kb, total_kb + 7):
            sp, kbps, last, stages = diag._wgrad_geometry(total_kb, req)
            assert (sp - 1) * kbps + last == total_kb and 1 <= last <= kbps and sp <= max(1, req)
            assert stages == min(4, kbps)
        pick = diag._one_kb_last(total_kb)
        if pick is not None:
            sp, kbps, last, _ = diag._wgrad_geometry(total_kb, pick)
            assert last == 1 and kbps > 1 and sp >= 3
    assert diag._one_kb_last(196) == 16 and diag._one_kb_last(448) is not None


def test_bound_sees_one_missing_k_block(diag, capsys):
    """At M = 802,816 rows (ResNet-50 layer 1 at batch 256) the result rounded to fp32 passes the bound, and the same
    result without one 64-row K-block fails it on most elements."""
    x, dy = _operands(256, 8, 56, 56, 8, (1, 1), 1, (0, 0), 1, seed=4)
    ref = diag._wgrad_ref64(x, dy, (1, 1), 1, 0)
    s2 = diag._wgrad_ref64(x, dy, (1, 1), 1, 0, squares=True)
    g0 = (torch.randn(ref.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
          * ref.pow(2).mean().sqrt()).float().double()
    assert diag._wgrad_check("exact sum", (g0 + ref).float(), g0, ref, s2, 132, "t") < 1.0
    assert diag.RESULTS[-1]
    rows = torch.arange(x.shape[0] * 56 * 56).view(x.shape[0], 56, 56)
    dropped = ((rows >= 64 * 5000) & (rows < 64 * 5001)).to(torch.float64).unsqueeze(1)
    partial = diag._wgrad_ref64(x, dy * (1 - dropped), (1, 1), 1, 0)
    diag._wgrad_check("one K-block missing", (g0 + partial).float(), g0, ref, s2, 132, "t")
    assert not diag.RESULTS[-1]
    line = [l for l in capsys.readouterr().out.splitlines() if "one K-block missing" in l][-1]
    bad = int(line.split("violations=")[1].split("/")[0])
    assert bad > ref.numel() // 2, line
    assert diag.WGRAD_C <= 2.0 ** -10
