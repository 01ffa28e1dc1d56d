"""MobileNetV2 on CPU: torchvision parity (state_dict, parameter counts, forward, gradients, running statistics), the
ReLU6 composites, the depthwise support predicate, and the compiled depthwise / ReLU6 BN kernels (ptxas)."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F
import torchvision

from distributeddeeplearning_b200 import _ext, models, ops
from distributeddeeplearning_b200.ops import native

# the 17 depthwise layers of MobileNetV2 as (C, H=W of the input, stride)
DW_SHAPES = [(32, 112, 1), (96, 112, 2), (144, 56, 1), (144, 56, 2), (192, 28, 1), (192, 28, 1), (192, 28, 2),
             (384, 14, 1), (384, 14, 1), (384, 14, 1), (384, 14, 1), (576, 14, 1), (576, 14, 1), (576, 14, 2),
             (960, 7, 1), (960, 7, 1), (960, 7, 1)]


@pytest.mark.parametrize("width", [1.0, 0.5])
def test_state_dict_and_param_count_match_torchvision(width):
    m = models.get_model("mobilenet_v2", width_mult=width)
    tv = torchvision.models.mobilenet_v2(width_mult=width)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in tv.state_dict().items()}
    n = sum(p.numel() for p in m.parameters())
    assert n == sum(p.numel() for p in tv.parameters())
    if width == 1.0:
        assert n == 3_504_872
    assert models.input_size("mobilenet_v2") == 224


def test_depthwise_layers_are_the_table():
    m = models.get_model("mobilenet_v2")
    got, hw = [], 112
    for blk in m.features[1:18]:
        dw = blk.conv[-3][0]
        assert dw.groups == dw.in_channels == dw.out_channels and tuple(dw.weight.shape[1:]) == (1, 3, 3)
        got.append((dw.in_channels, hw, dw.stride))
        hw = (hw - 1) // dw.stride + 1
    assert got == DW_SHAPES


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m = models.get_model("mobilenet_v2")
    bn = m.features[1].conv[0][1]
    assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))
    fc = m.classifier[1]
    assert torch.equal(fc.bias, torch.zeros_like(fc.bias)) and abs(float(fc.weight.detach().std()) - 0.01) < 1e-3
    w = m.features[5].conv[1][0].weight         # depthwise [192, 1, 3, 3]: kaiming normal, fan_out = 192 * 9
    assert abs(float(w.detach().std()) - (2.0 / (192 * 9)) ** 0.5) < 0.1 * (2.0 / (192 * 9)) ** 0.5
    assert w.is_contiguous(memory_format=torch.channels_last)


def test_mobilenet_v2_forward_backward_equals_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("mobilenet_v2"), torchvision.models.mobilenet_v2()
    m.load_state_dict(tv.state_dict())
    tv = tv.double()          # small batches make BN backward ill-conditioned: compare against float64
    m.train(), tv.train()
    m.classifier[0].p = tv.classifier[0].p = 0.0      # dropout masks come from different generators
    x = torch.randn(4, 3, 96, 96)
    y = torch.tensor([1, 7, 3, 9])
    o1, o2 = m(x), tv(x.double())
    assert torch.allclose(o1.double(), o2, atol=5e-4, rtol=1e-3)
    ops.softmax_cross_entropy(o1, y).backward()
    F.cross_entropy(o2, y).backward()
    g1, g2 = dict(m.named_parameters()), dict(tv.named_parameters())
    for k, p in g2.items():
        # floor: the beta gradient of a BN whose output feeds conv + BN is zero up to rounding (the next BN removes
        # any shift)
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-4))
        assert err < 5e-2, (k, err)
    assert tuple(g1["features.2.conv.1.0.weight"].grad.shape) == (96, 1, 3, 3)
    for k in ("features.0.1", "features.1.conv.0.1", "features.4.conv.1.1", "features.14.conv.3", "features.18.1"):
        a, b = m.get_submodule(k), tv.get_submodule(k)
        assert torch.allclose(a.running_mean.double(), b.running_mean, atol=1e-5), k
        assert torch.allclose(a.running_var.double(), b.running_var, atol=1e-5, rtol=1e-4), k


def test_mobilenet_v2_eval_equals_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("mobilenet_v2", num_classes=10), torchvision.models.mobilenet_v2(num_classes=10)
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    x = torch.randn(2, 3, 64, 80)
    with torch.no_grad():
        assert torch.allclose(m(x), tv(x), atol=1e-4, rtol=1e-4)


def test_relu6_composites_equal_relu6_of_batch_norm():
    torch.manual_seed(0)
    x = torch.randn(3, 16, 9, 7) * 4
    w = torch.randn(16, 16, 3, 3) * 0.5
    g, b = torch.rand(16) + 0.5, torch.randn(16) * 3
    for training in (True, False):
        rm1, rv1 = torch.randn(16) * 0.1, torch.rand(16) + 0.5
        rm2, rv2 = rm1.clone(), rv1.clone()
        z = ops.conv_bn_act(x, w, g, b, rm1, rv1, 1, 1, training=training, relu6=True)
        ref = F.relu6(F.batch_norm(F.conv2d(x, w, None, 1, 1), rm2, rv2, g, b, training))
        assert torch.allclose(z, ref, atol=1e-5, rtol=1e-5)
        assert float(z.max()) == 6.0 and float(z.min()) == 0.0      # the inputs straddle both clamp points
        assert torch.allclose(rm1, rm2) and torch.allclose(rv1, rv2)
        rm1, rv1 = torch.randn(16) * 0.1, torch.rand(16) + 0.5
        rm2, rv2 = rm1.clone(), rv1.clone()
        z = ops.batch_norm_act(x, g, b, rm1, rv1, training=training, relu6=True)
        assert torch.allclose(z, F.relu6(F.batch_norm(x, rm2, rv2, g, b, training)), atol=1e-5, rtol=1e-5)
    # depthwise composite (CPU) with ReLU6 and the defaults unchanged
    wd = torch.randn(16, 1, 3, 3)
    rm, rv = torch.zeros(16), torch.ones(16)
    z = ops.conv_bn_act(x, wd, g, b, rm, rv, 2, 1, groups=16, relu6=True)
    ref = F.relu6(F.batch_norm(F.conv2d(x, wd, None, 2, 1, 1, 16), torch.zeros(16), torch.ones(16), g, b, True))
    assert torch.allclose(z, ref, atol=1e-5, rtol=1e-5)
    z = ops.conv_bn_act(x, w, g, b, rm, rv, 1, 1)
    assert float(z.max()) > 6.0


def test_supports_depthwise_predicate():
    for c, _, s in DW_SHAPES:
        assert native.supports_depthwise(c, (3, 3), s, 1, 1, c), (c, s)
    assert native.supports_depthwise(8, 3, 1, (1, 1), 1, 8)
    assert native.supports_depthwise(40, (3, 3), 2, 1, 1, 40)
    assert not native.supports_depthwise(36, (3, 3), 1, 1, 1, 36)       # C % 8 != 0
    assert not native.supports_depthwise(32, (5, 5), 1, 2, 1, 32)       # 5x5
    assert not native.supports_depthwise(32, (3, 3), 3, 1, 1, 32)       # stride 3
    assert not native.supports_depthwise(32, (3, 3), 1, 2, 2, 32)       # dilation 2
    assert not native.supports_depthwise(32, (3, 3), 1, 0, 1, 32)       # padding 0
    assert not native.supports_depthwise(64, (3, 3), 1, 1, 1, 16)       # grouped, not depthwise
    assert not native.supports_depthwise(64, (3, 3), 1, 1, 1, 1)        # dense
    assert not native.supports_grouped(128, 128, 128)                    # the grouped predicate is unchanged


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
def test_depthwise_kernels_compile_without_spills():
    k = {n: v for n, v in _ptxas("depthwise.cu").items() if "dwconv_" in n}
    assert len(k) == 8, sorted(k)          # fwd (stride 1/2 x stats), dgrad and wgrad (stride 1/2)
    for name, (regs, st, ld) in k.items():
        assert st == 0 and ld == 0 and regs <= 128, (name, regs, st, ld)   # 2 blocks of 256 threads per SM


# (registers, spill stores, spill loads) of the BN kernels of the ResNet path with CUDA 12.9, before ReLU6 was added:
# the ReLU6 instantiations must leave them as they were.  MASK: 0 none, 1 z, 2 x, 3 bit mask.
BN_PARENT = {"bn_act_fwd_kernel<false, false, false, false>": (58, 0, 0),
             "bn_act_fwd_kernel<false, true, false, false>": (59, 0, 0),
             "bn_act_fwd_kernel<true, false, false, false>": (56, 0, 0),
             "bn_act_fwd_kernel<true, false, true, false>": (59, 0, 0),
             "bn_act_fwd_kernel<true, true, false, false>": (60, 0, 0),
             "bn_act_fwd_kernel<true, true, true, false>": (62, 0, 0),
             "bn_act_bwd_reduce_kernel<0>": (53, 0, 0), "bn_act_bwd_reduce_kernel<1>": (58, 0, 0),
             "bn_act_bwd_reduce_kernel<2>": (64, 0, 0), "bn_act_bwd_reduce_kernel<3>": (55, 0, 0),
             "bn_act_bwd_apply_kernel<0, false, false>": (64, 0, 0), "bn_act_bwd_apply_kernel<0, false, true>": (64, 0, 0),
             "bn_act_bwd_apply_kernel<0, true, false>": (56, 0, 0), "bn_act_bwd_apply_kernel<0, true, true>": (64, 0, 0),
             "bn_act_bwd_apply_kernel<1, false, false>": (64, 0, 0), "bn_act_bwd_apply_kernel<1, false, true>": (64, 0, 0),
             "bn_act_bwd_apply_kernel<1, true, false>": (56, 0, 0), "bn_act_bwd_apply_kernel<1, true, true>": (64, 0, 0),
             "bn_act_bwd_apply_kernel<2, false, false>": (64, 0, 0), "bn_act_bwd_apply_kernel<2, false, true>": (64, 8, 8),
             "bn_act_bwd_apply_kernel<2, true, false>": (64, 0, 0), "bn_act_bwd_apply_kernel<2, true, true>": (64, 4, 4),
             "bn_act_bwd_apply_kernel<3, false, false>": (64, 0, 0), "bn_act_bwd_apply_kernel<3, false, true>": (64, 0, 0),
             "bn_act_bwd_apply_kernel<3, true, false>": (56, 0, 0), "bn_act_bwd_apply_kernel<3, true, true>": (64, 0, 0)}


@pytest.mark.skipif(not _NVCC, reason="needs nvcc and c++filt")
def test_bn_kernels_keep_registers_and_relu6_has_no_spills():
    k = _ptxas("bn_act.cu")
    short = {re.sub(r"^void ddl::|\(ddl::Bn\w+Args\)$", "", n): tuple(v) for n, v in k.items()}
    assert {n: short.get(n) for n in BN_PARENT} == BN_PARENT
    relu6 = [n for n in short if n.endswith(", true>") and n.startswith("bn_act_fwd") or re.search(r"<[45][,>]", n)]
    assert len(relu6) == 10, relu6         # fwd train / eval x flat / chunked; reduce and apply (no fp8) of masks z6, x6
    for n in relu6:
        assert short[n][1:] == (0, 0), (n, short[n])
