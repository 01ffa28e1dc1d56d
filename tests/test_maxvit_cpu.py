"""MaxViT-T on CPU: torchvision parity (state_dict keys, order, shapes and dtypes, the parameter count, unsupported
builder arguments, stochastic-depth probabilities, initialisation, eval logits at 224 and 448, and train-mode logits,
every parameter gradient and the input gradient against float64 with the same stochastic-depth draws), the grid
attention and attention-layer composites against torchvision's modules in float64, the grid row map and bias index,
the predicates and the new kernels' ptxas figures."""
import re

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.models.maxvit import MaxVit as TvMaxVit
from torchvision.models.maxvit import PartitionAttentionLayer as TvLayer
from torchvision.models.maxvit import RelativePositionalMultiHeadAttention as TvAttn
from torchvision.models.maxvit import SwapAxes, WindowDepartition, WindowPartition
from torchvision.ops.stochastic_depth import StochasticDepth

from distributeddeeplearning_b200 import models, ops
from distributeddeeplearning_b200.models.maxvit import PartitionAttentionLayer
from distributeddeeplearning_b200.ops import native

from test_vit_cpu import _NVCC, _ptxas

PARAMS = 30_919_624


def test_state_dict_order_shapes_dtypes_and_parameter_count_match_torchvision():
    m, tv = models.get_model("maxvit_t"), torchvision.models.maxvit_t()
    a, b = m.state_dict(), tv.state_dict()
    assert list(a) == list(b) and len(a) == 582
    assert [(tuple(v.shape), v.dtype) for v in a.values()] == [(tuple(v.shape), v.dtype) for v in b.values()]
    assert [k for k, _ in m.named_parameters()] == [k for k, _ in tv.named_parameters()]
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == PARAMS
    idx = [k for k in a if k.endswith("relative_position_index")]
    assert len(idx) == 22 and all(torch.equal(a[k], b[k]) for k in idx)
    assert len([k for k in a if k.endswith("num_batches_tracked")]) == 34
    bns = [mod for mod in m.modules() if isinstance(mod, models.layers.BatchNorm2d)]
    assert bns and all(bn.eps == 1e-3 and bn.momentum == 0.01 for bn in bns)
    assert all(ln.eps == 1e-5 for ln in m.modules() if isinstance(ln, models.layers.LayerNorm))
    assert models.input_size(m) == models.input_size("maxvit_t") == 224


def test_builder_arguments_input_size_and_stochastic_depth():
    m = models.get_model("maxvit_t", num_classes=10, stochastic_depth_prob=0.4, input_size=448)
    assert m.classifier[5].out_features == 10 and m.input_size == 448
    layers = [ly for b in m.blocks for ly in b.layers]
    want = pytest.approx([0.4 * i / 10 for i in range(11)])
    assert [ly.layers["MBconv"].sd_prob for ly in layers] == want
    assert [ly.layers["grid_attention"].sd_prob for ly in layers] == want
    for kw in (dict(mlp_dropout=0.1), dict(attention_dropout=0.1), dict(pretrained=True), dict(input_size=256),
               dict(input_size=160)):
        with pytest.raises(ValueError):
            models.get_model("maxvit_t", **kw)


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("maxvit_t"), torchvision.models.maxvit_t()
    tvd = tv.state_dict()
    for k, p in m.state_dict().items():
        q = tvd[k]
        if k.endswith(("relative_position_index", "num_batches_tracked", "running_mean", "running_var")):
            assert torch.equal(p, q), k
        elif p.dim() == 1 and (k.endswith("weight") and ("norm" in k or re.search(r"(conv_[ab]|stem\.0)\.1\.", k)
                                                        or re.search(r"(attn|mlp)_layer\.0\.", k)
                                                        or k.startswith("classifier.2"))):
            assert torch.equal(p, torch.ones_like(p)) and torch.equal(q, p), k
        elif p.dim() == 1:
            assert torch.equal(p, torch.zeros_like(p)) and torch.equal(q, p), k
        else:                                # normal / trunc_normal, std 0.02: the same spread as torchvision's draw
            tol = 0.02 + 4 / p.numel() ** 0.5
            assert abs(float(p.std()) / float(q.std()) - 1) < tol and abs(float(p.std()) / 0.02 - 1) < tol, k
    assert m.stem[0][0].weight.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("size", [224, 448])
def test_eval_equals_torchvision(size):
    torch.manual_seed(size)
    m = models.get_model("maxvit_t", num_classes=10, input_size=size)
    tv = torchvision.models.maxvit_t(num_classes=10, input_size=(size, size))
    with torch.no_grad():
        for p in tv.parameters():
            p.add_(torch.randn_like(p) * 0.02)
        for mod in tv.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.5, 1.5)
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    x = torch.randn(1 if size == 448 else 2, 3, size, size)
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
                        else x * replay.pop(0).view(-1, *([1] * (x.dim() - 1))).to(x.dtype))
    return keeps, replay


def test_train_forward_backward_equals_float64_torchvision_with_the_same_stochastic_depth(monkeypatch):
    torch.manual_seed(3)
    m = models.get_model("maxvit_t", stochastic_depth_prob=0.5)
    tv = TvMaxVit((224, 224), 64, 7, [64, 128, 256, 512], [2, 2, 5, 2], 32, 0.5)   # maxvit_t's builder fixes p
    with torch.no_grad():
        for name, p in tv.named_parameters():
            if p.dim() == 1 or name.startswith("classifier"):
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
    assert not replay and len(keeps) == 50      # MBConv one, each attention layer two, in every layer but the first
    assert sum(int((k == 0).sum()) for k in keeps) > 0
    assert torch.allclose(o1.double(), o2, atol=1e-3, rtol=1e-3), float((o1.double() - o2).abs().max())
    ops.softmax_cross_entropy(o1, y).backward()
    F.cross_entropy(o2, y).backward()
    g1 = dict(m.named_parameters())
    for k, p in tv.named_parameters():
        if k.endswith("pre_norm.bias"):      # zero in exact arithmetic (a train-mode BN follows the 1x1 conv)
            assert float(p.grad.norm()) < 1e-12 and float(g1[k].grad.norm()) < 1e-5, k
            continue
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-6))
        assert err < 1e-3, (k, err)
    assert float(g1["blocks.0.layers.0.layers.grid_attention.attn_layer.1.relative_position_bias_table"].grad
                 .abs().max()) > 0
    err = float((xs.grad.double() - xd.grad).norm() / xd.grad.norm())
    assert err < 1e-3, err


def _tv_attention(x, attn, partition):
    """torchvision's partition -> (swap) -> attention (with merge) -> (swap) -> departition on [B, C, H, W]."""
    H, W = x.shape[2], x.shape[3]
    p = 7 if partition == "window" else H // 7
    t = WindowPartition()(x, p)
    if partition == "grid":
        t = SwapAxes(-2, -3)(t)
    t = attn(t)
    if partition == "grid":
        t = SwapAxes(-2, -3)(t)
    return WindowDepartition()(t, p, H // p, W // p)


@pytest.mark.parametrize("H", [7, 14, 28, 56])
def test_grid_attention_composite_equals_torchvision_in_float64(H):
    """ops.grid_attention on the qkv rows against torchvision's grid partition + attention (merge = identity)."""
    torch.manual_seed(H)
    C, heads = 64, 2
    attn = TvAttn(C, 32, 49).double()
    with torch.no_grad():
        attn.merge.weight.copy_(torch.eye(C))
        attn.merge.bias.zero_()
        attn.relative_position_bias_table.normal_()
    x = torch.randn(2, C, H, H, dtype=torch.float64)
    ref = _tv_attention(x, attn, "grid")
    qkv = F.linear(x.permute(0, 2, 3, 1), attn.to_qkv.weight, attn.to_qkv.bias).reshape(-1, 3 * C)
    out = ops.grid_attention(qkv, attn.relative_position_bias_table, heads, H, H)
    assert torch.allclose(out.view(2, H, H, C).permute(0, 3, 1, 2), ref, atol=1e-10, rtol=1e-10)


@pytest.mark.parametrize("partition", ["window", "grid"])
@pytest.mark.parametrize("H,sd", [(7, False), (14, True), (28, False), (56, True)])
def test_attention_layer_composite_equals_torchvision_in_float64(monkeypatch, partition, H, sd):
    torch.manual_seed(H + len(partition))
    C = 64
    p = 0.5 if sd else 0.0
    ref = TvLayer(C, 32, 7, partition, (H, H), 4, torch.nn.GELU, torch.nn.LayerNorm, 0.0, 0.0, p).double()
    with torch.no_grad():
        for q in ref.parameters():
            q.add_(torch.randn_like(q) * 0.2)
    layer = PartitionAttentionLayer(C, partition, p).double()
    layer.load_state_dict(ref.state_dict())
    assert list(layer.state_dict()) == list(ref.state_dict())
    keeps, replay = _record_replay(monkeypatch)
    x = torch.randn(3, C, H, H, dtype=torch.float64, requires_grad=True)
    xr = x.detach().clone().requires_grad_(True)
    z = layer(x)
    replay[:] = keeps
    zr = ref(xr)
    assert len(keeps) == (2 if sd else 0) and not replay
    assert torch.allclose(z, zr, atol=1e-10, rtol=1e-10)
    g = torch.randn_like(zr)
    z.backward(g)
    zr.backward(g)
    assert torch.allclose(x.grad, xr.grad, atol=1e-10, rtol=1e-10)
    for (k, a), (_, b) in zip(layer.named_parameters(), ref.named_parameters()):
        assert torch.allclose(a.grad, b.grad, atol=1e-10, rtol=1e-10), k


def test_grid_row_map_and_bias_index_match_torchvision():
    """The kernels' token -> pixel maps (grid: (a p + i, b p + j); window: (7 i + a, 7 j + b)) and the bias index
    (a - a' + 6) * 13 + (b - b' + 6) against torchvision's partition ops and relative_position_index."""
    for H in (7, 14, 28, 56):
        pix = torch.arange(H * H, dtype=torch.float64).view(1, 1, H, H)
        p = H // 7
        for partition in ("grid", "window"):
            q = 7 if partition == "window" else p
            t = WindowPartition()(pix, q)
            if partition == "grid":
                t = SwapAxes(-2, -3)(t)
            seq = t.reshape(-1, 49).long()                        # [sequences, 49] pixel of every token
            i, j = torch.div(torch.arange(seq.shape[0]), H // 7, rounding_mode="floor"), torch.arange(seq.shape[0]) % (H // 7)
            a, b = torch.arange(49) // 7, torch.arange(49) % 7
            if partition == "grid":
                y, x = a[None] * p + i[:, None], b[None] * p + j[:, None]
            else:
                y, x = 7 * i[:, None] + a[None], 7 * j[:, None] + b[None]
            assert torch.equal(seq, y * H + x), (H, partition)
    tv_idx = TvAttn(64, 32, 49).relative_position_index
    a, b = torch.arange(49) // 7, torch.arange(49) % 7
    idx = (a[:, None] - a[None] + 6) * 13 + (b[:, None] - b[None] + 6)
    assert torch.equal(idx, tv_idx)


def test_tvattention_scale_is_the_channel_count():
    """torchvision scales k by feat_dim^-1/2 (C, not the head dim): the kernels take it as a runtime scale."""
    assert TvAttn(256, 32, 49).scale_factor == 256 ** -0.5


def test_predicates_and_refusals():
    assert native.supports_grid_attention(56, 56, 7, 2, 32) and native.supports_grid_attention(7, 7, 7, 16, 32)
    assert native.supports_grid_attention(112, 112, 7, 2, 32)
    assert not native.supports_grid_attention(14, 28, 7, 4, 32)       # non-square
    assert not native.supports_grid_attention(40, 40, 7, 2, 32)       # not a multiple of 7
    assert not native.supports_grid_attention(56, 56, 8, 2, 32)       # partition 8
    assert not native.supports_grid_attention(56, 56, 7, 2, 64)       # head dim 64
    assert not native.supports_grid_attention(56, 56, 7, 0, 32)
    assert not native.supports_grid_attention(56, 56, 7, 65536, 32)
    x = torch.randn(2, 16, 8, 8)
    w, g, b = torch.randn(16, 16, 1, 1), torch.ones(16), torch.zeros(16)
    rm, rv = torch.zeros(16), torch.ones(16)
    for kw in ({"residual": x}, {"silu": True}, {"relu6": True}, {"hardswish": True}):
        with pytest.raises(ValueError):
            ops.conv_bn_act(x, w, g, b, rm, rv, relu=False, gelu=True, **kw)
    z = ops.conv_bn_act(x, w, g, b, rm, rv, relu=False, gelu=True, training=False)
    assert torch.allclose(z, F.gelu(F.conv2d(x, w)), atol=1e-5)
    with pytest.raises(ValueError):
        ops.maxvit_attention_layer(x, "shifted", 1, 1e-5, *([None] * 13))
    y = torch.randn(4, 512)
    assert torch.equal(ops.maxvit.tanh(y), torch.tanh(y))


@pytest.mark.skipif(not _NVCC, reason="needs nvcc and c++filt")
def test_new_kernels_compile_without_spills_and_fit_their_launch_bounds():
    ga = _ptxas("window_attention.cu")
    # nvcc 12.9 register counts of the grid (true) and window (false) partition instances; Swin's instances and the
    # shared bias-gradient reduction are pinned in test_swin_cpu.py
    used = {n: v[0] for n, v in ga.items() if "Partition" in n}
    assert used == {"win_attn_fwd_kernel<ddl::Partition<true> >": 70, "win_attn_fwd_kernel<ddl::Partition<false> >": 66,
                    "win_attn_bwd_kernel<ddl::Partition<true> >": 168,
                    "win_attn_bwd_kernel<ddl::Partition<false> >": 168}, used
    for n, (regs, st, ld, stack) in ga.items():
        assert st == 0 and ld == 0 and stack == 0 and regs <= 255, (n, regs, st, ld, stack)   # 128 threads
    bn = _ptxas("bn_act.cu")
    new = [n for n in bn if n.startswith("bn_gelu_fwd_kernel") or re.search(r"<9[,>]", n)]
    assert len(new) == 7, sorted(new)      # fwd train / eval x flat / chunked; reduce and apply (flat / chunked)
    for n in new:
        assert bn[n][1:] == [0, 0, 0] and bn[n][0] <= 64, (n, bn[n])           # __launch_bounds__(256, 4)
    misc = {n: v for n, v in _ptxas("misc_ops.cu").items() if "tanh_rows" in n}
    assert sorted(misc) == ["tanh_rows_bwd_kernel", "tanh_rows_fwd_kernel"], sorted(misc)
    for n, (regs, st, ld, stack) in misc.items():
        assert st == 0 and ld == 0 and stack == 0, (n, regs, st, ld, stack)
