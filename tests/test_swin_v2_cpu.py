"""Swin-V2-T, -S and -B on CPU: torchvision parity (state_dict keys, order and shapes, parameter counts, buffers,
initialisation, builder arguments, input size, eval logits at 256 and at 224, where three stages pad, and swin_v2_t's
train-mode logits, every parameter gradient and the input gradient against float64 with the same stochastic-depth
draws), the block, attention and PatchMergingV2 composites against torchvision in float64, the index, mask and
coordinate formulas of the kernels, the predicates and the new kernels' ptxas figures."""
import math
import re

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.models.swin_transformer import PatchMergingV2 as TvMerge
from torchvision.models.swin_transformer import ShiftedWindowAttentionV2 as TvAttn
from torchvision.models.swin_transformer import SwinTransformer as TvSwin
from torchvision.models.swin_transformer import SwinTransformerBlockV2 as TvBlock
from torchvision.models.swin_transformer import shifted_window_attention

from distributeddeeplearning_b200 import models, ops
from distributeddeeplearning_b200.models.swin_v2 import PatchMergingV2, SwinTransformerBlockV2
from distributeddeeplearning_b200.ops import native
from distributeddeeplearning_b200.ops.swin_v2 import relative_coords_table

from test_swin_cpu import _record_replay
from test_vit_cpu import _NVCC, _ptxas

NAMES = ["swin_v2_t", "swin_v2_s", "swin_v2_b"]
PARAMS = dict(zip(NAMES, [28_351_570, 49_737_442, 87_930_848]))
KEYS = dict(zip(NAMES, [233, 449, 449]))


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_order_shapes_buffers_and_parameter_counts_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    sd, tsd = m.state_dict(), tv.state_dict()
    assert list(sd) == list(tsd) and len(sd) == KEYS[name]
    assert [tuple(v.shape) for v in sd.values()] == [tuple(v.shape) for v in tsd.values()]
    assert [k for k, _ in m.named_parameters()] == [k for k, _ in tv.named_parameters()]
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == PARAMS[name]
    assert models.input_size(m) == models.input_size(name) == 256
    for k, v in sd.items():
        if k.endswith("relative_position_index") or k.endswith("relative_coords_table"):
            assert v.dtype == tsd[k].dtype and torch.equal(v, tsd[k]), k
    assert sd["features.1.0.attn.relative_coords_table"].shape == (1, 15, 15, 2)
    assert sd["features.1.0.attn.relative_position_index"].shape == (4096,)
    assert all(ln.eps == 1e-5 for ln in m.modules() if isinstance(ln, models.layers.LayerNorm))
    for stage, s in enumerate((1, 3, 5, 7)):
        for b in m.features[s]:
            C = b.norm1.weight.numel()
            for Hs in (64 >> stage, 56 >> stage):             # 256 and 224 (28, 14 and 7 pad)
                assert native.supports_window_attention_v2(Hs, Hs, 8, b.attn.num_heads, C // b.attn.num_heads)
            assert native.supports_layer_norm(C)
    for pm in (m.features[2], m.features[4], m.features[6]):
        assert native.supports_layer_norm(pm.norm.weight.numel())


def test_builder_arguments_and_stochastic_depth():
    m = models.get_model("swin_v2_t", num_classes=10, stochastic_depth_prob=0.4)
    assert m.head.out_features == 10
    blocks = [b for s in (1, 3, 5, 7) for b in m.features[s]]
    assert [b.sd_prob for b in blocks] == pytest.approx([0.4 * i / 11 for i in range(12)])
    assert [b.attn.shift_size for b in blocks] == [0, 4] * 6 and all(b.attn.window_size == 8 for b in blocks)
    assert [b.attn.num_heads for b in blocks] == [3, 3, 6, 6] + [12] * 6 + [24, 24]
    assert [b.sd_prob for b in models.get_model("swin_v2_t").features[7]][-1] == pytest.approx(0.2)
    assert [b.sd_prob for b in models.get_model("swin_v2_s").features[7]][-1] == pytest.approx(0.3)
    d = models.get_model("swin_v2_b")
    assert [b.sd_prob for b in d.features[7]][-1] == pytest.approx(0.5)
    assert d.features[0][0].weight.shape[0] == 128 and [b.attn.num_heads for b in d.features[7]] == [32, 32]
    for kw in (dict(dropout=0.1), dict(attention_dropout=0.1), dict(pretrained=True)):
        with pytest.raises(ValueError):
            models.get_model("swin_v2_t", **kw)


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("swin_v2_t"), torchvision.models.swin_v2_t()
    for k, p in m.state_dict().items():
        q = tv.state_dict()[k]
        if k.endswith("relative_position_index") or k.endswith("relative_coords_table"):
            continue
        if k.endswith("logit_scale"):
            assert torch.equal(p, q) and torch.allclose(p, torch.full_like(p, math.log(10))), k
        elif re.search(r"norm\d?\.weight$", k) or k == "features.0.2.weight":
            assert torch.equal(p, torch.ones_like(p)), k
        elif (re.search(r"norm\d?\.bias$", k) or k == "features.0.2.bias" or k.endswith("mlp.0.bias")
              or k.endswith("mlp.3.bias") or k.endswith("qkv.bias") or k.endswith("proj.bias") or k == "head.bias"
              or k.endswith("cpb_mlp.0.bias")):
            assert torch.equal(p, torch.zeros_like(p)) and torch.equal(q, torch.zeros_like(q)), k
        else:                                # random: same spread (and range) as torchvision's draw, within sampling noise
            tol = 0.02 + 4 / p.numel() ** 0.5
            assert abs(float(p.std()) / float(q.std()) - 1) < tol, k
            assert abs(float(p.mean())) < tol * float(q.std()) + 1e-3 * (k == "features.0.0.bias"), k
    a = m.features[1][0].attn
    for p in (a.cpb_mlp[0].weight, a.cpb_mlp[2].weight, m.features[1][0].mlp[0].weight):   # trunc_normal(0.02)
        assert abs(float(p.detach().std()) / 0.02 - 1) < 0.15


@pytest.mark.parametrize("size", [256, 224])
def test_eval_equals_torchvision(size):
    torch.manual_seed(size)
    m, tv = models.get_model("swin_v2_t", num_classes=10), torchvision.models.swin_v2_t(num_classes=10)
    with torch.no_grad():
        for p in tv.parameters():
            p.add_(torch.randn_like(p) * 0.02)       # perturbed norms, biases (k-bias too: ignored by both) and head
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    x = torch.randn(2, 3, size, size)
    with torch.no_grad():
        out, ref = m(x), tv(x)
    assert torch.allclose(out, ref, atol=1e-4, rtol=1e-4), float((out - ref).abs().max())


@pytest.mark.parametrize("size", [224])
def test_swin_v2_t_train_forward_backward_equals_float64_torchvision_with_the_same_stochastic_depth(monkeypatch, size):
    torch.manual_seed(3)
    m = models.get_model("swin_v2_t", stochastic_depth_prob=0.5)
    tv = TvSwin([4, 4], 96, [2, 2, 6, 2], [3, 6, 12, 24], [8, 8], stochastic_depth_prob=0.5, block=TvBlock,
                downsample_layer=TvMerge)
    with torch.no_grad():
        for name, p in tv.named_parameters():
            if p.dim() == 1 or name.startswith("head"):
                p.add_(torch.randn_like(p) * 0.1)
    m.load_state_dict(tv.state_dict())
    tv = tv.double()
    m.train(), tv.train()
    keeps, replay = _record_replay(monkeypatch)
    x = torch.randn(2, 3, size, size)
    xs, xd = x.clone().requires_grad_(True), x.double().requires_grad_(True)
    y = torch.tensor([1, 7])
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
        if k.endswith("qkv.bias"):
            C = p.numel() // 3
            assert torch.equal(p.grad[C:2 * C], torch.zeros_like(p.grad[C:2 * C])), k
            assert torch.equal(g1[k].grad[C:2 * C], torch.zeros_like(g1[k].grad[C:2 * C])), k
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-6))
        assert err < 1e-3, (k, err)
    for k in ("features.1.0.attn.logit_scale", "features.1.0.attn.cpb_mlp.0.weight", "features.1.0.attn.cpb_mlp.2.weight",
              "features.5.0.attn.qkv.bias"):
        assert float(g1[k].grad.abs().max()) > 0, k
    err = float((xs.grad.double() - xd.grad).norm() / xd.grad.norm())
    assert err < 1e-3, err


@pytest.mark.parametrize("shift,H,W,sd", [(0, 16, 16, False), (4, 16, 24, False), (4, 16, 16, True), (4, 8, 16, True),
                                          (4, 14, 14, True), (4, 7, 20, False), (0, 10, 12, True)])
def test_block_composite_equals_torchvision_in_float64(monkeypatch, shift, H, W, sd):
    torch.manual_seed(shift + H + W)
    C, heads = 64, 2
    ref = TvBlock(C, heads, [8, 8], [shift, shift], stochastic_depth_prob=0.5 if sd else 0.0).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(torch.randn_like(p) * 0.2)
    blk = SwinTransformerBlockV2(C, heads, 8, shift, 0.5 if sd else 0.0).double()
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
    assert torch.equal(blk.attn.qkv.bias.grad[C:2 * C], torch.zeros(C, dtype=torch.float64))


@pytest.mark.parametrize("H,W", [(16, 16), (7, 10)])
def test_patch_merging_v2_composite_equals_torchvision_in_float64(H, W):
    torch.manual_seed(H * W)
    C = 16
    ref = TvMerge(C).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(torch.randn_like(p) * 0.2)
    pm = PatchMergingV2(C).double()
    pm.load_state_dict(ref.state_dict())
    assert list(pm.state_dict()) == list(ref.state_dict()) == ["reduction.weight", "norm.weight", "norm.bias"]
    assert tuple(pm.norm.weight.shape) == (2 * C,)
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


@pytest.mark.parametrize("H,W,shift,clamp", [(16, 16, 4, False), (16, 32, 4, False), (8, 16, 4, False),
                                             (8, 8, 4, False), (24, 16, 0, False), (14, 14, 4, False),
                                             (7, 20, 4, False), (10, 12, 4, True)])
def test_window_attention_v2_composite_equals_torchvision_in_float64(H, W, shift, clamp):
    """ops.window_attention_v2 on the qkv rows (k-bias zeroed, as torchvision does) against torchvision's
    shifted_window_attention with logit_scale, its qkv bias and an identity proj, with every gradient: padded maps carry
    q = b_q, k = 0, v = b_v on the padding tokens."""
    torch.manual_seed(H + W + shift)
    C, heads = 64, 2
    x = torch.randn(2, H, W, C, dtype=torch.float64)
    wq = torch.randn(3 * C, C, dtype=torch.float64) * C ** -0.5
    bq = torch.randn(3 * C, dtype=torch.float64, requires_grad=True)
    table = (torch.rand(225, heads, dtype=torch.float64) * 16).requires_grad_(True)
    ls = torch.log(10 * torch.ones(heads, 1, 1, dtype=torch.float64))
    if clamp:
        ls[0] = 5.0                                                   # above ln 100: clamped, gradient 0
    ls.requires_grad_(True)
    idx = ops.swin.relative_position_index(8)
    bias = table[idx].view(64, 64, -1).permute(2, 0, 1).contiguous().unsqueeze(0)
    ref = shifted_window_attention(x, wq, torch.eye(C, dtype=torch.float64), bias, [8, 8], heads, [shift, shift],
                                   qkv_bias=bq, logit_scale=ls, training=False)
    g = torch.randn_like(ref)
    gr = torch.autograd.grad(ref, (bq, table, ls), g)
    b2 = bq.detach().clone().requires_grad_(True)
    t2, l2 = table.detach().clone().requires_grad_(True), ls.detach().clone().requires_grad_(True)
    beff = torch.cat([b2[:C], torch.zeros(C, dtype=torch.float64), b2[2 * C:]])
    out = ops.window_attention_v2(F.linear(x, wq, beff).reshape(-1, 3 * C), t2, l2, b2[:C], b2[2 * C:], heads, H, W, 8,
                                  shift)
    assert torch.allclose(out.view(2, H, W, C), ref, atol=1e-10, rtol=1e-10)
    go = torch.autograd.grad(out.view(2, H, W, C), (b2, t2, l2), g)
    for a, b in zip(go, gr):
        assert torch.allclose(a, b, atol=1e-10, rtol=1e-10)
    assert torch.equal(go[0][C:2 * C], torch.zeros(C, dtype=torch.float64))
    if clamp:
        assert float(go[2][0]) == 0.0 and float(go[2][1]) != 0.0


def test_relative_index_padded_mask_and_coords_formulas_match_torchvision():
    """The kernels' analytic index (iy - jy + 7) * 15 + (ix - jx + 7), the regions computed on the padded frame, and the
    relative_coords_table formula, against torchvision's tensors."""
    tva = TvAttn(32, [8, 8], [0, 0], 1)
    i = torch.arange(64)
    iy, ix = i // 8, i % 8
    idx = (iy[:, None] - iy[None, :] + 7) * 15 + (ix[:, None] - ix[None, :] + 7)
    assert torch.equal(idx.flatten(), tva.relative_position_index)
    assert torch.equal(ops.swin.relative_position_index(8), tva.relative_position_index)
    assert torch.equal(relative_coords_table(8), tva.relative_coords_table)
    for H, W, s in ((64, 64, 4), (28, 28, 4), (14, 14, 4), (7, 7, 4), (8, 20, 4), (20, 36, 4), (56, 56, 0)):
        sy, sx = native.window_shift(H, W, 8, s)
        pH, pW = -(-H // 8) * 8, -(-W // 8) * 8
        if sy + sx == 0:
            assert (pH == 8 or pW == 8 or s == 0)
            continue
        mask = torch.zeros(pH, pW)
        count = 0
        for h in ((0, -8), (-8, -sy), (-sy, None)):
            for w in ((0, -8), (-8, -sx), (-sx, None)):
                mask[h[0]:h[1], w[0]:w[1]] = count
                count += 1
        mask = mask.view(pH // 8, 8, pW // 8, 8).permute(0, 2, 1, 3).reshape(-1, 64)
        tv_m = (mask.unsqueeze(1) - mask.unsqueeze(2)) != 0
        y, x = torch.arange(pH), torch.arange(pW)
        by = torch.where(y < pH - 8, 0, torch.where(y < pH - sy, 1, 2))
        bx = torch.where(x < pW - 8, 0, torch.where(x < pW - sx, 1, 2))
        reg = (3 * by[:, None] + bx[None, :]).view(pH // 8, 8, pW // 8, 8).permute(0, 2, 1, 3).reshape(-1, 64)
        assert torch.equal(reg[:, :, None] != reg[:, None, :], tv_m), (H, W, s)


def test_predicates():
    for H in (64, 32, 16, 8, 56, 28, 14, 7, 5, 20):
        assert native.supports_window_attention_v2(H, H, 8, 3, 32)
    assert native.supports_window_attention_v2(20, 36, 8, 32, 32)
    assert not native.supports_window_attention_v2(64, 64, 7, 3, 32)     # window 7: Swin V1
    assert not native.supports_window_attention_v2(64, 64, 8, 3, 64)     # head dim 64
    assert not native.supports_window_attention_v2(64, 64, 8, 33, 32)    # more heads than the CPB kernels take
    assert not native.supports_window_attention_v2(64, 64, 8, 0, 32)
    assert not native.supports_window_attention_v2(0, 64, 8, 3, 32)
    assert native.window_shift(64, 64, 8, 4) == (4, 4) and native.window_shift(7, 7, 8, 4) == (0, 0)
    assert native.window_shift(8, 8, 8, 4) == (0, 0) and native.window_shift(14, 14, 8, 4) == (4, 4)
    assert native.window_shift(8, 20, 8, 4) == (0, 4)
    for C in (192, 384, 768, 256, 512, 1024):                            # the LayerNorm over 2C of PatchMergingV2
        assert native.supports_layer_norm(C)


@pytest.mark.skipif(not _NVCC, reason="needs nvcc and c++filt")
def test_new_kernels_compile_without_spills_and_fit_their_launch_bounds():
    wa = _ptxas("window_attention_v2.cu")
    used = {n: v[0] for n, v in wa.items()}     # nvcc 12.9
    assert used == {"win2_attn_fwd_kernel": 80, "win2_attn_bwd_kernel": 166, "mma_tile::grad_chunk_kernel<128, 64>": 26,
                    "win2_grad_final_kernel": 26}, used
    for n, (regs, st, ld, stack) in wa.items():
        assert st == 0 and ld == 0 and stack == 0 and regs <= 255, (n, regs, st, ld, stack)   # 128 threads
    sw = _ptxas("swin_v2.cu")
    assert sorted(sw) == ["cpb_bwd_kernel", "cpb_bwd_reduce_kernel", "cpb_fwd_kernel", "merge_gather_kernel<false>",
                          "merge_gather_kernel<true>"], sorted(sw)
    for n, (regs, st, ld, stack) in sw.items():
        assert st == 0 and ld == 0 and stack == 0 and regs <= 255, (n, regs, st, ld, stack)   # <= 256 threads
