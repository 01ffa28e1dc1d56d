"""RegNetX / RegNetY on CPU: torchvision parity (state_dict, parameter counts, initialisation, eval logits and
train-mode gradients), the block composite against torchvision's ResBottleneckBlock, the group-bundle predicates and
operand layout of the grouped conv kernels, and the compiled conv kernels' ptxas figures."""
import os
import sys

import pytest
import torch
import torchvision
from torchvision.models.regnet import ResBottleneckBlock as TvBlock

from distributeddeeplearning_b200 import models, ops
from distributeddeeplearning_b200.models import regnet
from distributeddeeplearning_b200.ops import native

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_vit_cpu import _NVCC, _ptxas  # noqa: E402

PARAMS = {"regnet_x_400mf": 5_495_976, "regnet_x_800mf": 7_259_656, "regnet_x_1_6gf": 9_190_136,
          "regnet_x_3_2gf": 15_296_552, "regnet_x_8gf": 39_572_648, "regnet_x_16gf": 54_278_536,
          "regnet_x_32gf": 107_811_560, "regnet_y_400mf": 4_344_144, "regnet_y_800mf": 6_432_512,
          "regnet_y_1_6gf": 11_202_430, "regnet_y_3_2gf": 19_436_338, "regnet_y_8gf": 39_381_472,
          "regnet_y_16gf": 83_590_140, "regnet_y_32gf": 145_046_770, "regnet_y_128gf": 644_812_894}


@pytest.mark.parametrize("name", sorted(PARAMS))
def test_state_dict_and_param_count_match_torchvision(name):
    m = models.get_model(name)
    a = m.state_dict()
    del m
    tv = getattr(torchvision.models, name)()
    b = tv.state_dict()
    assert list(a) == list(b)
    assert all(tuple(a[k].shape) == tuple(b[k].shape) and a[k].dtype == b[k].dtype for k in a)
    assert sum(v.numel() for k, v in a.items() if "running" not in k and "num_batches" not in k) == PARAMS[name]
    assert sum(p.numel() for p in tv.parameters()) == PARAMS[name]


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m = models.get_model("regnet_y_800mf")
    for k in ("stem.0.weight", "trunk_output.block2.block2-1.f.a.0.weight", "trunk_output.block3.block3-0.f.b.0.weight",
              "trunk_output.block3.block3-0.f.se.fc1.weight", "trunk_output.block3.block3-0.f.se.fc2.weight",
              "trunk_output.block4.block4-0.proj.0.weight"):
        w = m.get_parameter(k).detach()
        want = (2.0 / (w.shape[0] * w.shape[2] * w.shape[3])) ** 0.5        # fan_out = k*k*out_channels
        assert abs(float(w.std()) / want - 1) < 0.05, (k, float(w.std()), want)
    fc1 = m.get_submodule("trunk_output.block3.block3-0.f.se.fc1")
    bound = 1 / fc1.weight.shape[1] ** 0.5                                   # nn.Conv2d's default bias init
    b = fc1.bias.detach()
    assert float(b.abs().max()) <= bound and float(b.std()) > 0.3 * bound
    assert abs(float(m.fc.weight.detach().std()) / 0.01 - 1) < 0.05 and float(m.fc.bias.detach().abs().max()) == 0.0
    bn = m.get_submodule("trunk_output.block1.block1-0.f.b.1")
    assert bn.eps == 1e-5 and bn.momentum == 0.1
    assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))


@pytest.mark.parametrize("name", ["regnet_x_400mf", "regnet_y_400mf"])
def test_eval_logits_match_torchvision(name):
    torch.manual_seed(0)
    tv = getattr(torchvision.models, name)()
    m = models.get_model(name)
    with torch.no_grad():                    # non-trivial running statistics
        for mod in tv.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.5, 1.5)
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.double().eval()
    x = torch.randn(2, 3, 224, 224)
    with torch.no_grad():
        o1, o2 = m(x), tv(x.double())
    assert torch.allclose(o1.double(), o2, atol=1e-4, rtol=1e-3), float((o1.double() - o2).abs().max())


def test_regnet_y_400mf_train_gradients_match_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("regnet_y_400mf"), torchvision.models.regnet_y_400mf()
    m.load_state_dict(tv.state_dict())
    tv = tv.double()          # small batches make BN backward ill-conditioned: compare against float64
    m.train(), tv.train()
    x = torch.randn(4, 3, 96, 96)
    xd = x.double().requires_grad_(True)
    x.requires_grad_(True)
    y = torch.tensor([1, 7, 3, 9])
    o1, o2 = m(x), tv(xd)
    assert torch.allclose(o1.double(), o2, atol=5e-4, rtol=1e-3)
    ops.softmax_cross_entropy(o1, y).backward()
    torch.nn.functional.cross_entropy(o2, y).backward()
    g1 = dict(m.named_parameters())
    for k, p in tv.named_parameters():
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-4))
        assert err < 5e-2, (k, err)
    err = float((x.grad.double() - xd.grad).norm() / xd.grad.norm())
    assert err < 5e-2, err


@pytest.mark.parametrize("win,wout,stride,cg,se", [(48, 48, 1, 16, False), (48, 72, 2, 24, False),
                                                   (48, 48, 1, 8, True), (232, 464, 2, 232, True)])
def test_block_composite_matches_torchvision(win, wout, stride, cg, se):
    """X / Y blocks, identity and projection, stride 2; Y's squeeze widths 12 and 58 are not multiples of 8."""
    torch.manual_seed(0)
    blk = regnet.ResBottleneckBlock(win, wout, stride, cg, 0.25 if se else None).train()
    tv = TvBlock(win, wout, stride, torch.nn.BatchNorm2d, torch.nn.ReLU, cg, 1.0, 0.25 if se else None)
    tv.load_state_dict(blk.state_dict())
    tv = tv.double().train()
    x = torch.randn(3, win, 9, 9, requires_grad=True)
    xd = x.detach().double().requires_grad_(True)
    o1, o2 = blk(x), tv(xd)
    assert torch.allclose(o1.double(), o2, atol=1e-5, rtol=1e-4)
    g = torch.randn(o2.shape, dtype=torch.float64)
    o1.backward(g.float())
    o2.backward(g)
    assert torch.allclose(x.grad.double(), xd.grad, atol=1e-4, rtol=1e-3)
    g1 = dict(blk.named_parameters())
    for k, p in tv.named_parameters():
        assert torch.allclose(g1[k].grad.double(), p.grad, atol=1e-4, rtol=1e-3), k
    if se:
        assert blk.f.se.fc1.out_channels == round(0.25 * win)


def test_grouped_predicates():
    shapes = regnet.grouped_shapes()
    assert len(shapes) == 101
    assert sorted({g for *_, g in shapes}) == [8, 16, 24, 48, 56, 112, 120, 128, 168, 232, 264]
    assert all(native.grouped_conv_native(c, c, c // g) for c, _, _, g in shapes)
    for c, cg in ((128, 4), (256, 8), (512, 16), (1024, 32), (2048, 64), (256, 4), (512, 8), (2048, 32)):
        assert native.grouped_conv_native(c, c, c // cg) and native.supports_grouped(c, c, c // cg)
    assert not native.grouped_conv_native(96, 96, 96)             # depthwise
    assert not native.grouped_conv_native(128, 64, 32)            # Cin != Cout
    assert not native.grouped_conv_native(72, 72, 18)             # cg = 4 with C not a multiple of 64
    assert not native.grouped_conv_native(100, 100, 4)            # C % 8 != 0
    assert not native.grouped_conv_native(128, 128, 1)
    # supports_grouped keeps its truth table: the whole-groups-per-tile subset
    assert not native.supports_grouped(72, 72, 3) and not native.supports_grouped(448, 448, 4)
    assert native.supports_grouped(128, 128, 32) and not native.supports_grouped(96, 96, 3)


@pytest.mark.parametrize("cg,wb,t", [(8, 64, 1), (16, 64, 1), (24, 48, 1), (48, 48, 1), (56, 56, 1), (112, 112, 2),
                                     (128, 128, 2), (264, 264, 5)])
def test_bundle_geometry(cg, wb, t):
    assert native.grouped_bundle(cg) == (wb, t)


@pytest.mark.parametrize("C,cg", [(128, 4), (256, 8), (512, 16), (1024, 32), (2048, 64), (128, 64)])
def test_bundle_layout_is_the_resnext_layout_at_wb_64(C, cg):
    w = torch.randn(C, 9 * cg)
    e = native.expand_grouped_weight_ref(w, 9, C // cg)
    ref = torch.zeros(C, 9 * 64)
    co = torch.arange(C)
    for tap in range(9):
        for j in range(cg):
            ref[co, tap * 64 + (co % 64 - co % cg) + j] = w[:, tap * cg + j]
    assert torch.equal(e, ref)


@pytest.mark.parametrize("C,cg", [(72, 24), (48, 8), (528, 264), (448, 56), (224, 112)])
def test_bundle_layout_rows_and_zero_overhang(C, cg):
    taps = 9
    wb, t = native.grouped_bundle(cg)
    w = torch.randn(C, taps * cg)
    e = native.expand_grouped_weight_ref(w, taps, C // cg)
    assert tuple(e.shape) == native.grouped_expanded_shape(C, taps, C // cg) == (-(-C // wb) * t * 64, taps * t * 64)
    for co in range(C):
        b, l = divmod(co, wb)
        row = e[b * t * 64 + l].view(taps, t * 64)
        g0 = l - l % cg
        assert torch.equal(row[:, g0:g0 + cg], w[co].view(taps, cg))
        assert int((row != 0).sum()) == int((w[co] != 0).sum())
    live = torch.zeros(e.shape[0], dtype=torch.bool)
    for co in range(C):
        live[co // wb * t * 64 + co % wb] = True
    assert int(e[~live].abs().sum()) == 0             # rows past Wb (and past C) are zero: dgrad's K overhang


def test_input_size_and_builder_arguments():
    assert models.input_size("regnet_y_16gf") == 224
    assert models.get_model("regnet_x_400mf", num_classes=10).fc.out_features == 10
    for kw in ({"norm_layer": None}, {"activation": None}, {"stem_type": None}, {"block_type": None}):
        with pytest.raises(ValueError):
            models.get_model("regnet_y_400mf", **kw)


# conv_gemm.cu ptxas figures at the parent commit, (registers, spill stores, spill loads, stack): the 64-wide
# instantiations that take grouped launches grow by one or two registers; nothing gains spills or stack.  (Ten of the
# 128-wide instantiations with BN statistics already spilled at the parent and are unchanged.)
PARENT_GROUPED = {"conv_gemm_kernel<64, 4, false, 0, false, false>": 70, "conv_gemm_kernel<64, 4, true, 0, false, false>": 74,
                  "conv_gemm_kernel<64, 5, false, 0, false, false>": 70, "conv_gemm_kernel<64, 5, true, 0, false, false>": 74,
                  "conv_gemm_kernel<64, 0, true, 0, false, false>": 96, "conv_gemm_kernel<64, 1, true, 0, false, false>": 96,
                  "conv_wgrad_kernel<4, true>": 58, "conv_wgrad_kernel<0, true>": 58}
PARENT_SPILLS = {"conv_gemm_kernel<128, 0, true, 0, false, false>": 28, "conv_gemm_kernel<128, 1, true, 0, false, false>": 28,
                 "conv_gemm_kernel<128, 2, true, 0, false, false>": 8, "conv_gemm_kernel<128, 2, true, 0, true, false>": 8,
                 "conv_gemm_kernel<128, 2, true, 0, true, true>": 28, "conv_gemm_kernel<128, 2, true, 1, false, false>": 20,
                 "conv_gemm_kernel<128, 3, true, 0, false, false>": 28, "conv_gemm_kernel<128, 6, true, 0, false, false>": 8,
                 "conv_gemm_kernel<128, 6, true, 0, true, false>": 8, "conv_gemm_kernel<128, 6, true, 0, true, true>": 28,
                 "conv_gemm_kernel<128, 6, true, 2, false, false>": 20}


@pytest.mark.skipif(not _NVCC, reason="nvcc / c++filt not available")
def test_conv_gemm_ptxas_no_new_spills():
    k = _ptxas("conv_gemm.cu")
    assert len(k) == 91, sorted(k)
    for n, (regs, st, ld, stack) in k.items():
        if n in PARENT_SPILLS:
            assert st <= PARENT_SPILLS[n] and ld <= PARENT_SPILLS[n], (n, regs, st, ld, stack)
        else:
            assert st == 0 and ld == 0 and stack == 0, (n, regs, st, ld, stack)
    for n, regs in PARENT_GROUPED.items():
        assert k[n][0] <= regs + 4, (n, k[n], regs)
