"""MobileNetV3-Large / -Small on CPU: torchvision parity (state_dict, parameter counts, depthwise tables, initialisation,
forward, gradients, running statistics), the hardswish and squeeze-excitation composites, the 5x5 depthwise support
predicate, and the compiled 5x5 depthwise / hardswish BN / squeeze-excitation kernels (ptxas)."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.ops import SqueezeExcitation

from distributeddeeplearning_b200 import _ext, models, ops
from distributeddeeplearning_b200.models.mobilenet import _make_divisible
from distributeddeeplearning_b200.models.mobilenetv3 import ConvBNAct, SqueezeExcitation as SE
from distributeddeeplearning_b200.ops import native

# depthwise layers as (C, H=W of the input, kernel, stride)
DW_LARGE = [(16, 112, 3, 1), (64, 112, 3, 2), (72, 56, 3, 1), (72, 56, 5, 2), (120, 28, 5, 1), (120, 28, 5, 1),
            (240, 28, 3, 2), (200, 14, 3, 1), (184, 14, 3, 1), (184, 14, 3, 1), (480, 14, 3, 1), (672, 14, 3, 1),
            (672, 14, 5, 2), (960, 7, 5, 1), (960, 7, 5, 1)]
DW_SMALL = [(16, 112, 3, 2), (72, 56, 3, 2), (88, 28, 3, 1), (96, 28, 5, 2), (240, 14, 5, 1), (240, 14, 5, 1),
            (120, 14, 5, 1), (144, 14, 5, 1), (288, 14, 5, 2), (576, 7, 5, 1), (576, 7, 5, 1)]
PARAMS = {"mobilenet_v3_large": 5_483_032, "mobilenet_v3_small": 2_542_856}
NAMES = ["mobilenet_v3_large", "mobilenet_v3_small"]


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("width", [1.0, 0.75])
def test_state_dict_and_param_count_match_torchvision(name, width):
    m = models.get_model(name, width_mult=width)
    tv = getattr(torchvision.models, name)(width_mult=width)
    assert list(m.state_dict()) == list(tv.state_dict())
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in tv.state_dict().items()}
    n = sum(p.numel() for p in m.parameters())
    assert n == sum(p.numel() for p in tv.parameters())
    if width == 1.0:
        assert n == PARAMS[name]
    assert models.input_size(name) == 224 and m.input_size == 224
    for mod in m.modules():
        if hasattr(mod, "running_var"):
            assert mod.eps == 1e-3 and mod.momentum == 0.01


def _dw_and_se(m):
    dws, ses, hw = [], [], 112
    for blk in m.features[1:-1]:
        for mod in blk.block:
            if isinstance(mod, ConvBNAct) and mod[0].groups > 1:
                c, k, s = mod[0].in_channels, mod[0].kernel_size[0], mod[0].stride
                assert mod[0].groups == c == mod[0].out_channels and mod[0].padding == k // 2
                dws.append((c, hw, k, s))
                hw = (hw - 1) // s + 1
            elif isinstance(mod, SE):
                ses.append((mod.fc1.in_channels, mod.fc1.out_channels))
    return dws, ses


@pytest.mark.parametrize("name,table,n_se", [("mobilenet_v3_large", DW_LARGE, 8), ("mobilenet_v3_small", DW_SMALL, 9)])
def test_depthwise_and_se_layers_are_the_table(name, table, n_se):
    dws, ses = _dw_and_se(models.get_model(name))
    assert dws == table
    assert len(ses) == n_se
    for c, cs in ses:
        assert c % 8 == 0 and cs == _make_divisible(c // 4, 8) and cs % 8 == 0, (c, cs)


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m = models.get_model("mobilenet_v3_large")
    bn = m.features[1].block[0][1]
    assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))
    for fc in (m.classifier[0], m.classifier[3]):
        assert torch.equal(fc.bias, torch.zeros_like(fc.bias)) and abs(float(fc.weight.detach().std()) - 0.01) < 1e-3
    se = m.features[4].block[2]
    assert isinstance(se, SE)
    for conv in (se.fc1, se.fc2):
        assert torch.equal(conv.bias, torch.zeros_like(conv.bias))        # torchvision zero-initialises conv biases
    w = m.features[5].block[1][0].weight           # depthwise [120, 1, 5, 5]: kaiming normal, fan_out = 120 * 25
    assert tuple(w.shape) == (120, 1, 5, 5)
    ref = (2.0 / (120 * 25)) ** 0.5
    assert abs(float(w.detach().std()) - ref) < 0.1 * ref
    assert w.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("name", NAMES)
def test_forward_backward_equals_torchvision(name):
    torch.manual_seed(0)
    m, tv = models.get_model(name), getattr(torchvision.models, name)()
    m.load_state_dict(tv.state_dict())
    tv = tv.double()          # small batches make BN backward ill-conditioned: compare against float64
    m.train(), tv.train()
    m.classifier[2].p = tv.classifier[2].p = 0.0      # dropout masks come from different generators
    x = torch.randn(4, 3, 96, 96)
    y = torch.tensor([1, 7, 3, 9])
    o1, o2 = m(x), tv(x.double())
    assert torch.allclose(o1.double(), o2, atol=5e-4, rtol=1e-3)
    ops.softmax_cross_entropy(o1, y).backward()
    F.cross_entropy(o2, y).backward()
    g1, g2 = dict(m.named_parameters()), dict(tv.named_parameters())
    for k, p in g2.items():
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-4))
        assert err < 5e-2, (k, err)
    for k, mod in m.named_modules():
        if hasattr(mod, "running_mean"):
            b = tv.get_submodule(k)
            assert torch.allclose(mod.running_mean.double(), b.running_mean, atol=1e-5), k
            assert torch.allclose(mod.running_var.double(), b.running_var, atol=1e-5, rtol=1e-4), k


@pytest.mark.parametrize("name", NAMES)
def test_eval_equals_torchvision(name):
    torch.manual_seed(0)
    m, tv = models.get_model(name, num_classes=10), getattr(torchvision.models, name)(num_classes=10)
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    x = torch.randn(2, 3, 64, 80)
    with torch.no_grad():
        assert torch.allclose(m(x), tv(x), atol=1e-4, rtol=1e-4)


def test_hardswish_composites_equal_hardswish_of_batch_norm():
    torch.manual_seed(0)
    x = torch.randn(3, 16, 9, 7) * 4
    w = torch.randn(16, 16, 3, 3) * 0.5
    g, b = torch.rand(16) + 0.5, torch.randn(16) * 3
    for training in (True, False):
        rm1, rv1 = torch.randn(16) * 0.1, torch.rand(16) + 0.5
        rm2, rv2 = rm1.clone(), rv1.clone()
        z = ops.conv_bn_act(x, w, g, b, rm1, rv1, 1, 1, training=training, hardswish=True)
        v = F.batch_norm(F.conv2d(x, w, None, 1, 1), rm2, rv2, g, b, training)
        assert torch.allclose(z, F.hardswish(v), atol=1e-5, rtol=1e-5)
        assert float((v < -3).float().mean()) > 0.05 and float((v > 3).float().mean()) > 0.05     # straddles both
        assert torch.allclose(rm1, rm2) and torch.allclose(rv1, rv2)
    # depthwise 5x5 composite (CPU) with hardswish, and the refusals
    wd = torch.randn(16, 1, 5, 5)
    rm, rv = torch.zeros(16), torch.ones(16)
    z = ops.conv_bn_act(x, wd, g, b, rm, rv, 2, 2, groups=16, hardswish=True)
    ref = F.hardswish(F.batch_norm(F.conv2d(x, wd, None, 2, 2, 1, 16), torch.zeros(16), torch.ones(16), g, b, True))
    assert torch.allclose(z, ref, atol=1e-5, rtol=1e-5)
    with pytest.raises(ValueError):
        ops.conv_bn_act(x, w, g, b, rm, rv, 1, 1, residual=x, hardswish=True)
    with pytest.raises(ValueError):
        ops.conv_bn_act(x, w, g, b, rm, rv, 1, 1, relu6=True, hardswish=True)
    h = torch.linspace(-5, 5, 101)
    assert torch.equal(ops.hardswish(h), F.hardswish(h))


@pytest.mark.parametrize("c,cs", [(16, 8), (72, 24), (960, 240)])
def test_squeeze_excite_equals_torchvision(c, cs):
    torch.manual_seed(0)
    ref = SqueezeExcitation(c, cs, scale_activation=torch.nn.Hardsigmoid).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(torch.randn_like(p) * 0.5)
    w1, b1, w2, b2 = (p.detach().clone().requires_grad_(True) for p in
                      (ref.fc1.weight, ref.fc1.bias, ref.fc2.weight, ref.fc2.bias))
    x = (torch.randn(3, c, 5, 6, dtype=torch.float64) * 3).requires_grad_(True)
    xr = x.detach().clone().requires_grad_(True)
    y = ops.squeeze_excite(x, w1, b1, w2, b2)
    yr = ref(xr)
    assert torch.allclose(y, yr, atol=1e-12, rtol=1e-12)
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g)
    assert torch.allclose(x.grad, xr.grad, atol=1e-12, rtol=1e-10)
    for got, p in zip((w1, b1, w2, b2), (ref.fc1.weight, ref.fc1.bias, ref.fc2.weight, ref.fc2.bias)):
        assert torch.allclose(got.grad, p.grad, atol=1e-12, rtol=1e-10)


def test_supports_depthwise5_predicate():
    """The 5x5 kernels have their own predicate; the 3x3 one keeps its scope (5x5 stays outside it)."""
    for c, _, k, s in DW_LARGE + DW_SMALL:
        assert native.depthwise_native(c, (k, k), s, k // 2, 1, c), (c, k, s)
        assert native.supports_depthwise5(c, (k, k), s, k // 2, 1, c) == (k == 5), (c, k, s)
        assert native.supports_depthwise(c, (k, k), s, k // 2, 1, c) == (k == 3), (c, k, s)
    assert native.supports_depthwise5(8, 5, 2, (2, 2), 1, 8)
    assert native.supports_depthwise5(32, (5, 5), 1, 2, 1, 32)
    assert not native.supports_depthwise5(32, (5, 5), 1, 1, 1, 32)      # 5x5 with padding 1
    assert not native.supports_depthwise5(32, (3, 3), 1, 1, 1, 32)      # 3x3 (the other family)
    assert not native.supports_depthwise5(36, (5, 5), 1, 2, 1, 36)      # C % 8 != 0
    assert not native.supports_depthwise5(32, (5, 5), 3, 2, 1, 32)      # stride 3
    assert not native.supports_depthwise5(32, (5, 5), 1, 4, 2, 32)      # dilation 2
    assert not native.supports_depthwise5(32, (7, 7), 1, 3, 1, 32)      # 7x7
    assert not native.supports_depthwise5(32, (3, 5), 1, (1, 2), 1, 32)  # rectangular
    assert not native.supports_depthwise5(64, (5, 5), 1, 2, 1, 16)      # grouped, not depthwise
    assert not native.depthwise_native(32, (7, 7), 1, 3, 1, 32) and not native.depthwise_native(32, (3, 3), 1, 2, 1, 32)


def _ptxas(src):
    """{demangled kernel name: (registers, spill store bytes, spill load bytes)} of one .cu file built for sm_90a."""
    nvcc = os.path.join(_ext.CUDA_HOME, "bin", "nvcc")
    csrc = os.path.join(os.path.dirname(_ext.__file__), "csrc")
    r = subprocess.run([nvcc, "-c", os.path.join(csrc, "ops", src), "-o", os.devnull, "-O3", "-std=c++17", *_ext.NVCC_ARCH,
                        "--expt-relaxed-constexpr", "-I", csrc, "-Xptxas", "-v"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            cur = cur.replace("(anonymous namespace)::", "")
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = [0, int(m.group(1)), int(m.group(2))]
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            out[cur][0] = int(m.group(1))
    return out


_NVCC = shutil.which("c++filt") and os.path.isfile(os.path.join(_ext.CUDA_HOME, "bin", "nvcc"))


@pytest.mark.skipif(not _NVCC, reason="needs nvcc and c++filt")
def test_new_kernels_compile_without_spills_and_fit_their_launch_bounds():
    k = {n: v for n, v in _ptxas("depthwise5.cu").items() if "dwconv5_" in n}
    assert len(k) == 8, sorted(k)          # fwd (stride 1/2 x stats), dgrad and wgrad (stride 1/2)
    for name, (regs, st, ld) in k.items():
        assert st == 0 and ld == 0 and regs <= 80, (name, regs, st, ld)    # __launch_bounds__(256, 3)
    bn = {re.sub(r"^void ddl::|\(ddl::Bn\w+Args\)$", "", n): tuple(v) for n, v in _ptxas("bn_act.cu").items()}
    hs = [n for n in bn if n.startswith("bn_hswish_fwd_kernel") or re.search(r"<6[,>]", n)]
    assert len(hs) == 7, hs                # fwd train / eval x flat / chunked; reduce and apply (flat / chunked)
    for n in hs:
        assert bn[n][1:] == (0, 0) and bn[n][0] <= 64, (n, bn[n])         # __launch_bounds__(256, 4)
    se = {n: v for n, v in _ptxas("squeeze_excite.cu").items() if "se_" in n}
    assert len(se) == 3, sorted(se)
    misc = {n: v for n, v in _ptxas("misc_ops.cu").items() if "hardswish" in n}
    assert len(misc) == 2, sorted(misc)
    for name, (regs, st, ld) in list(se.items()) + list(misc.items()):
        assert st == 0 and ld == 0, (name, regs, st, ld)
