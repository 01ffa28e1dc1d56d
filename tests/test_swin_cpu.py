"""Swin-T, -S and -B on CPU: torchvision parity (state_dict keys, order and shapes, parameter counts, the relative position
index, unsupported builder arguments, initialisation, eval logits at 224 and at a size that needs padding, and swin_t's
train-mode logits, every parameter gradient and the input gradient against float64 with the same stochastic-depth
draws), the block, patch-merging and window-attention composites against torchvision in float64, the predicates and
the new kernels' ptxas figures."""
import re

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.models.swin_transformer import PatchMerging as TvPatchMerging
from torchvision.models.swin_transformer import SwinTransformer as TvSwin
from torchvision.models.swin_transformer import SwinTransformerBlock as TvBlock
from torchvision.models.swin_transformer import shifted_window_attention
from torchvision.ops.stochastic_depth import StochasticDepth

from distributeddeeplearning_b200 import models, ops
from distributeddeeplearning_b200.models.swin import PatchMerging, SwinTransformerBlock
from distributeddeeplearning_b200.ops import native

from test_vit_cpu import _NVCC, _ptxas

NAMES = ["swin_t", "swin_s", "swin_b"]
PARAMS = dict(zip(NAMES, [28_288_354, 49_606_258, 87_768_224]))


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_order_shapes_index_and_parameter_counts_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    assert list(m.state_dict()) == list(tv.state_dict())
    assert [tuple(v.shape) for v in m.state_dict().values()] == [tuple(v.shape) for v in tv.state_dict().values()]
    assert [k for k, _ in m.named_parameters()] == [k for k, _ in tv.named_parameters()]
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == PARAMS[name]
    assert models.input_size(m) == models.input_size(name) == 224
    for k, v in m.state_dict().items():
        if k.endswith("relative_position_index"):
            assert v.dtype == torch.int64 and torch.equal(v, tv.state_dict()[k]), k
    lns = [mod for mod in m.modules() if isinstance(mod, models.layers.LayerNorm)]
    assert all(ln.eps == 1e-5 for ln in lns)
    for stage, (Hs, blocks) in enumerate(zip((56, 28, 14, 7), (m.features[1], m.features[3], m.features[5],
                                                               m.features[7]))):
        for b in blocks:
            C = b.norm1.weight.numel()
            assert native.supports_window_attention(Hs, Hs, 7, b.attn.num_heads, C // b.attn.num_heads)
            assert native.supports_layer_norm(C)
    for pm in (m.features[2], m.features[4], m.features[6]):
        C = pm.norm.weight.numel() // 4
        assert native.supports_patch_merge(56, 56, C)


def test_unsupported_builder_arguments_and_stochastic_depth():
    m = models.get_model("swin_t", num_classes=10, stochastic_depth_prob=0.4)
    assert m.head.out_features == 10
    blocks = [b for s in (1, 3, 5, 7) for b in m.features[s]]
    assert [b.sd_prob for b in blocks] == pytest.approx([0.4 * i / 11 for i in range(12)])
    assert [b.attn.shift_size for b in blocks] == [0, 3] * 6
    d = models.get_model("swin_b")
    assert [b.sd_prob for s in (1, 3, 5, 7) for b in d.features[s]][-1] == pytest.approx(0.5)
    for kw in (dict(dropout=0.1), dict(attention_dropout=0.1), dict(pretrained=True)):
        with pytest.raises(ValueError):
            models.get_model("swin_t", **kw)


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("swin_t"), torchvision.models.swin_t()
    for k, p in m.state_dict().items():
        q = tv.state_dict()[k]
        if k.endswith("relative_position_index"):
            continue
        if re.search(r"norm\d?\.weight$", k) or k == "features.0.2.weight":
            assert torch.equal(p, torch.ones_like(p)), k
        elif (re.search(r"norm\d?\.bias$", k) or k == "features.0.2.bias" or k.endswith("mlp.0.bias")
              or k.endswith("mlp.3.bias") or k.endswith("qkv.bias") or k.endswith("proj.bias") or k == "head.bias"):
            assert torch.equal(p, torch.zeros_like(p)) and torch.equal(q, torch.zeros_like(q)), k
        else:                                # random: same spread (and range) as torchvision's draw, within sampling noise
            tol = 0.02 + 4 / p.numel() ** 0.5
            assert abs(float(p.std()) / float(q.std()) - 1) < tol, k
            assert abs(float(p.mean())) < tol * float(q.std()) + 1e-3 * (k == "features.0.0.bias"), k
    # trunc_normal(std 0.02): the bias table, and the MLP re-initialised by the model's final loop (not xavier: 0.064)
    for p in (m.features[1][0].attn.relative_position_bias_table, m.features[1][0].mlp[0].weight):
        assert abs(float(p.detach().std()) / 0.02 - 1) < 0.1
    assert m.features[0][0].weight.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("size", [224, 160])
def test_eval_equals_torchvision(size):
    torch.manual_seed(size)
    m, tv = models.get_model("swin_t", num_classes=10), torchvision.models.swin_t(num_classes=10)
    with torch.no_grad():
        for p in tv.parameters():
            p.add_(torch.randn_like(p) * 0.02)       # perturbed LayerNorm affines and biases, a non-zero head
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        out, ref = m(x), tv(x)
    assert torch.allclose(out, ref, atol=1e-4, rtol=1e-4), float((out - ref).abs().max())


def _record_replay(monkeypatch):
    keeps, draw = [], ops.stochastic_depth_keep

    def record(n, p, device):
        keeps.append(draw(n, p, device))
        return keeps[-1]

    monkeypatch.setattr(ops, "stochastic_depth_keep", record)
    replay = []
    monkeypatch.setattr(StochasticDepth, "forward",
                        lambda self, x: x if self.p == 0.0 or not self.training
                        else x * replay.pop(0).view(-1, 1, 1, 1).to(x.dtype))
    return keeps, replay


def test_swin_t_train_forward_backward_equals_float64_torchvision_with_the_same_stochastic_depth(monkeypatch):
    torch.manual_seed(3)
    m = models.get_model("swin_t", stochastic_depth_prob=0.5)
    tv = TvSwin([4, 4], 96, [2, 2, 6, 2], [3, 6, 12, 24], [7, 7], stochastic_depth_prob=0.5)   # swin_t's builder fixes p
    with torch.no_grad():
        for name, p in tv.named_parameters():
            if p.dim() == 1 or name.startswith("head"):
                p.add_(torch.randn_like(p) * 0.1)
    m.load_state_dict(tv.state_dict())
    tv = tv.double()
    m.train(), tv.train()
    keeps, replay = _record_replay(monkeypatch)
    x = torch.randn(4, 3, 224, 224)
    xs, xd = x.clone().requires_grad_(True), x.double().requires_grad_(True)
    y = torch.tensor([1, 7, 3, 9])
    o1 = m(xs)
    replay[:] = keeps
    o2 = tv(xd)
    assert not replay and len(keeps) == 22                  # two per block but the first (p = 0)
    assert sum(int((k == 0).sum()) for k in keeps) > 0
    assert torch.allclose(o1.double(), o2, atol=1e-3, rtol=1e-3), float((o1.double() - o2).abs().max())
    ops.softmax_cross_entropy(o1, y).backward()
    F.cross_entropy(o2, y).backward()
    g1 = dict(m.named_parameters())
    for k, p in tv.named_parameters():
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-6))
        assert err < 1e-3, (k, err)
    assert float(g1["features.1.0.attn.relative_position_bias_table"].grad.abs().max()) > 0
    err = float((xs.grad.double() - xd.grad).norm() / xd.grad.norm())
    assert err < 1e-3, err


@pytest.mark.parametrize("shift,H,W,sd", [(0, 14, 14, False), (3, 14, 21, False), (3, 14, 14, True), (3, 7, 14, True),
                                          (3, 10, 12, True)])
def test_block_composite_equals_torchvision_in_float64(monkeypatch, shift, H, W, sd):
    torch.manual_seed(shift + H + W)
    C, heads = 64, 2
    ref = TvBlock(C, heads, [7, 7], [shift, shift], stochastic_depth_prob=0.5 if sd else 0.0).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(torch.randn_like(p) * 0.2)
    blk = SwinTransformerBlock(C, heads, 7, shift, 0.5 if sd else 0.0).double()
    blk.load_state_dict(ref.state_dict())
    assert list(blk.state_dict()) == list(ref.state_dict())
    keeps, replay = _record_replay(monkeypatch)
    x = torch.randn(3, C, H, W, dtype=torch.float64, requires_grad=True)
    xr = x.detach().permute(0, 2, 3, 1).clone().requires_grad_(True)
    z = blk(x)
    replay[:] = keeps
    zr = ref(xr)
    assert len(keeps) == (2 if sd else 0) and not replay
    assert torch.allclose(z.permute(0, 2, 3, 1), zr, atol=1e-10, rtol=1e-10)
    g = torch.randn_like(zr)
    z.permute(0, 2, 3, 1).backward(g)
    zr.backward(g)
    assert torch.allclose(x.grad.permute(0, 2, 3, 1), xr.grad, atol=1e-10, rtol=1e-10)
    for (k, p), (_, q) in zip(blk.named_parameters(), ref.named_parameters()):
        assert torch.allclose(p.grad, q.grad, atol=1e-10, rtol=1e-10), k


@pytest.mark.parametrize("H,W", [(14, 14), (7, 10)])
def test_patch_merging_composite_equals_torchvision_in_float64(H, W):
    torch.manual_seed(H * W)
    C = 16
    ref = TvPatchMerging(C).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(torch.randn_like(p) * 0.2)
    pm = PatchMerging(C).double()
    pm.load_state_dict(ref.state_dict())
    assert list(pm.state_dict()) == list(ref.state_dict()) == ["reduction.weight", "norm.weight", "norm.bias"]
    x = torch.randn(2, C, H, W, dtype=torch.float64, requires_grad=True)
    xr = x.detach().permute(0, 2, 3, 1).clone().requires_grad_(True)
    z, zr = pm(x), ref(xr)
    assert torch.allclose(z.permute(0, 2, 3, 1), zr, atol=1e-10, rtol=1e-10)
    g = torch.randn_like(zr)
    z.permute(0, 2, 3, 1).backward(g)
    zr.backward(g)
    assert torch.allclose(x.grad.permute(0, 2, 3, 1), xr.grad, atol=1e-10, rtol=1e-10)
    for (k, p), (_, q) in zip(pm.named_parameters(), ref.named_parameters()):
        assert torch.allclose(p.grad, q.grad, atol=1e-10, rtol=1e-10), k


@pytest.mark.parametrize("H,W,shift", [(14, 14, 3), (14, 28, 3), (7, 14, 3), (7, 7, 3), (21, 14, 0), (10, 12, 3)])
def test_window_attention_composite_equals_torchvision_in_float64(H, W, shift):
    """ops.window_attention on the qkv rows against torchvision's shifted_window_attention with a bias-free qkv and an
    identity proj (padding included: a bias-free qkv of torchvision's zero padding is zero)."""
    torch.manual_seed(H + W + shift)
    C, heads = 64, 2
    x = torch.randn(2, H, W, C, dtype=torch.float64)
    wq = torch.randn(3 * C, C, dtype=torch.float64) * C ** -0.5
    table = torch.randn(169, heads, dtype=torch.float64)
    idx = ops.swin.relative_position_index(7)
    bias = table[idx].view(49, 49, -1).permute(2, 0, 1).contiguous().unsqueeze(0)
    ref = shifted_window_attention(x, wq, torch.eye(C, dtype=torch.float64), bias, [7, 7], heads, [shift, shift],
                                   training=False)
    out = ops.window_attention(F.linear(x, wq).reshape(-1, 3 * C), table, heads, H, W, 7, shift)
    assert torch.allclose(out.view(2, H, W, C), ref, atol=1e-10, rtol=1e-10)


def test_relative_position_index_and_mask_formulas_match_torchvision():
    """The kernels' analytic index (iy - jy + 6) * 13 + (ix - jx + 6) and regions against torchvision's tensors."""
    from torchvision.models.swin_transformer import ShiftedWindowAttention
    tv_idx = ShiftedWindowAttention(32, [7, 7], [0, 0], 1).relative_position_index
    i = torch.arange(49)
    iy, ix = i // 7, i % 7
    idx = (iy[:, None] - iy[None, :] + 6) * 13 + (ix[:, None] - ix[None, :] + 6)
    assert torch.equal(idx.flatten(), tv_idx) and torch.equal(ops.swin.relative_position_index(7), tv_idx)
    for H, W, s in ((56, 56, 3), (14, 28, 3), (7, 14, 3), (7, 14, 0)):
        sy, sx = native.window_shift(H, W, 7, s)
        if sy + sx == 0:
            continue
        mask = torch.zeros(H, W)
        count = 0
        for h in ((0, -7), (-7, -sy), (-sy, None)):
            for w in ((0, -7), (-7, -sx), (-sx, None)):
                mask[h[0]:h[1], w[0]:w[1]] = count
                count += 1
        mask = mask.view(H // 7, 7, W // 7, 7).permute(0, 2, 1, 3).reshape(-1, 49)
        tv_m = (mask.unsqueeze(1) - mask.unsqueeze(2)) != 0
        y = torch.arange(H)
        x = torch.arange(W)
        by = torch.where(y < H - 7, 0, torch.where(y < H - sy, 1, 2))
        bx = torch.where(x < W - 7, 0, torch.where(x < W - sx, 1, 2))
        reg = (3 * by[:, None] + bx[None, :]).view(H // 7, 7, W // 7, 7).permute(0, 2, 1, 3).reshape(-1, 49)
        assert torch.equal(reg[:, :, None] != reg[:, None, :], tv_m), (H, W, s)


def test_predicates():
    assert native.supports_window_attention(56, 56, 7, 3, 32) and native.supports_window_attention(7, 7, 7, 32, 32)
    assert native.supports_window_attention(14, 28, 7, 12, 32)
    assert not native.supports_window_attention(40, 40, 7, 3, 32)       # needs padding: the composite
    assert not native.supports_window_attention(56, 56, 7, 3, 64)       # head dim 64
    assert not native.supports_window_attention(64, 64, 8, 3, 32)       # window 8 (Swin V2)
    assert not native.supports_window_attention(56, 56, 7, 0, 32)
    assert native.window_shift(56, 56, 7, 3) == (3, 3) and native.window_shift(7, 7, 7, 3) == (0, 0)
    assert native.window_shift(7, 14, 7, 3) == (0, 3) and native.window_shift(5, 40, 7, 3) == (0, 3)
    for C in (96, 192, 384, 128, 256, 512):
        assert native.supports_patch_merge(56, 56, C)
    assert not native.supports_patch_merge(7, 7, 96) and not native.supports_patch_merge(56, 56, 1024)
    assert not native.supports_patch_merge(56, 56, 100)
    assert not native.supports_layer_norm(2048)                          # why patch merging has its own LayerNorm


@pytest.mark.skipif(not _NVCC, reason="needs nvcc and c++filt")
def test_new_kernels_compile_without_spills_and_fit_their_launch_bounds():
    wa = _ptxas("window_attention.cu")
    # nvcc 12.9 register counts of Swin's instances and the bias-gradient reduction; MaxViT's (Partition) are pinned
    # in test_maxvit_cpu.py
    used = {n: v[0] for n, v in wa.items() if "Partition" not in n}
    assert used == {"win_attn_fwd_kernel<ddl::ShiftedWindow>": 80, "win_attn_bwd_kernel<ddl::ShiftedWindow>": 255,
                    "mma_tile::grad_chunk_kernel<128, 64>": 26, "win_bias_grad_final_kernel": 25}, used
    for n, (regs, st, ld, stack) in wa.items():
        assert st == 0 and ld == 0 and stack == 0 and regs <= 255, (n, regs, st, ld, stack)   # 128 threads
    sw = _ptxas("swin.cu")
    assert len(sw) == 17, sorted(sw)          # merge fwd / bwd for K = 1..8 vectors per lane, the dgamma/dbeta reduce
    for n, (regs, st, ld, stack) in sw.items():
        assert st == 0 and ld == 0 and stack == 0 and regs <= 255, (n, regs, st, ld, stack)   # 256 threads
