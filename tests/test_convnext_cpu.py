"""ConvNeXt-Tiny to -Large on CPU: torchvision parity (state_dict, parameter counts, LayerNorm eps, stage widths and
depths, stochastic-depth probabilities, initialisation, eval logits, and convnext_tiny's train-mode logits, every
gradient and the input gradient against float64 with the same stochastic-depth draws), the block / LayerNorm / GELU /
layer-scale composites, the 7x7 depthwise predicate and the compiled kernels' ptxas figures."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.models.convnext import CNBlock as TvCNBlock, LayerNorm2d
from torchvision.ops import StochasticDepth

from distributeddeeplearning_b200 import _ext, models, ops
from distributeddeeplearning_b200.models.convnext import CNBlock
from distributeddeeplearning_b200.models.layers import LayerNorm
from distributeddeeplearning_b200.ops import native

NAMES = ["convnext_tiny", "convnext_small", "convnext_base", "convnext_large"]
PARAMS = dict(zip(NAMES, [28_589_128, 50_223_688, 88_591_464, 197_767_336]))
WIDTHS = dict(zip(NAMES, [(96, 192, 384, 768), (96, 192, 384, 768), (128, 256, 512, 1024), (192, 384, 768, 1536)]))
DEPTHS = dict(zip(NAMES, [(3, 3, 9, 3), (3, 3, 27, 3), (3, 3, 27, 3), (3, 3, 27, 3)]))
SD_P = dict(zip(NAMES, [0.1, 0.4, 0.5, 0.5]))


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_params_widths_eps_and_stochastic_depth_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    assert list(m.state_dict()) == list(tv.state_dict())
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in tv.state_dict().items()}
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == PARAMS[name]
    assert "features.1.0.block.2.weight" in m.state_dict() and "features.1.0.block.1.weight" not in m.state_dict()
    assert tuple(m.features[1][0].layer_scale.shape) == (WIDTHS[name][0], 1, 1)
    lns = [mod for mod in m.modules() if isinstance(mod, LayerNorm)]
    tvlns = [mod for mod in tv.modules() if isinstance(mod, torch.nn.LayerNorm)]
    assert len(lns) == len(tvlns) and all(a.eps == b.eps == 1e-6 for a, b in zip(lns, tvlns))
    stages = [m.features[i] for i in (1, 3, 5, 7)]
    assert tuple(len(s) for s in stages) == DEPTHS[name]
    assert tuple(s[0].block[0].in_channels for s in stages) == WIDTHS[name]
    blocks = [b for b in m.modules() if isinstance(b, CNBlock)]
    tvb = [b for b in tv.modules() if isinstance(b, TvCNBlock)]
    total = sum(DEPTHS[name])
    assert [b.sd_prob for b in blocks] == [b.stochastic_depth.p for b in tvb] == \
        [SD_P[name] * i / (total - 1.0) for i in range(total)]
    assert models.input_size(name) == m.input_size == 224
    for b in blocks:
        dw = b.block[0]
        assert native.supports_depthwise7(dw.in_channels, dw.kernel_size, dw.stride, dw.padding, dw.dilation, dw.groups)
        assert native.supports_layer_norm(dw.in_channels)
    with pytest.raises(ValueError):
        models.get_model(name, pretrained=True)


def test_builder_arguments_and_initialisation_follow_torchvision():
    torch.manual_seed(0)
    m = models.get_model("convnext_tiny", num_classes=10, stochastic_depth_prob=0.3, layer_scale=0.5)
    assert m.classifier[2].out_features == 10 and m.features[7][2].sd_prob == pytest.approx(0.3)
    assert torch.equal(m.features[1][0].layer_scale, torch.full((96, 1, 1), 0.5))
    m = models.get_model("convnext_base")
    assert torch.equal(m.features[5][4].layer_scale, torch.full((512, 1, 1), 1e-6))
    for w, b in ((m.features[0][0].weight, m.features[0][0].bias), (m.features[5][4].block[3].weight,
                 m.features[5][4].block[3].bias), (m.features[5][4].block[0].weight, m.features[5][4].block[0].bias),
                 (m.features[6][1].weight, m.features[6][1].bias), (m.classifier[2].weight, m.classifier[2].bias)):
        w = w.detach()
        assert torch.equal(b, torch.zeros_like(b))
        # trunc_normal_(std=0.02) truncates at +-2 (absolute): a normal of std 0.02, whose median |w| is 0.6745 * 0.02
        assert abs(float(w.abs().median()) - 0.6745 * 0.02) < 0.07 * 0.6745 * 0.02 and abs(float(w.mean())) < 0.002
    ln = m.features[6][0]
    assert torch.equal(ln.weight, torch.ones_like(ln.weight)) and torch.equal(ln.bias, torch.zeros_like(ln.bias))
    assert m.features[1][0].block[0].weight.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("name", NAMES)
def test_eval_equals_torchvision(name):
    torch.manual_seed(0)
    m, tv = models.get_model(name, num_classes=10), getattr(torchvision.models, name)(num_classes=10)
    with torch.no_grad():
        for p in tv.parameters():
            p.add_(torch.randn_like(p) * 0.05)       # non-trivial layer scales, LayerNorm affines and biases
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    x = torch.randn(2, 3, 64, 64)
    with torch.no_grad():
        out, ref = m(x), tv(x)
    assert torch.allclose(out, ref, atol=1e-4, rtol=1e-4), float((out - ref).abs().max())


def test_tiny_train_forward_backward_equals_float64_torchvision_with_the_same_stochastic_depth(monkeypatch):
    torch.manual_seed(3)
    m, tv = models.get_model("convnext_tiny", stochastic_depth_prob=0.5), torchvision.models.convnext_tiny(
        stochastic_depth_prob=0.5)
    with torch.no_grad():
        for name, p in tv.named_parameters():
            if name.endswith("layer_scale"):
                p.copy_(torch.rand_like(p) * 0.5 + 0.25)        # at 1e-6 a dropped or mis-scaled branch would not show
            elif p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.1)
    m.load_state_dict(tv.state_dict())
    tv = tv.double()
    m.train(), tv.train()
    keeps, draw = [], ops.stochastic_depth_keep

    def record(n, p, device):
        keeps.append(draw(n, p, device))
        return keeps[-1]

    monkeypatch.setattr(ops, "stochastic_depth_keep", record)
    replay = []
    monkeypatch.setattr(StochasticDepth, "forward",
                        lambda self, x: x if self.p == 0.0 else x * replay.pop(0).view(-1, 1, 1, 1).to(x.dtype))
    x = torch.randn(4, 3, 64, 64)
    xs, xd = x.clone().requires_grad_(True), x.double().requires_grad_(True)
    y = torch.tensor([1, 7, 3, 9])
    o1 = m(xs)
    replay[:] = keeps
    o2 = tv(xd)
    assert not replay and len(keeps) == 17                  # every block but the first (p = 0)
    assert sum(int((k == 0).sum()) for k in keeps) > 0
    assert torch.allclose(o1.double(), o2, atol=1e-3, rtol=1e-3), float((o1.double() - o2).abs().max())
    ops.softmax_cross_entropy(o1, y).backward()
    F.cross_entropy(o2, y).backward()
    g1, g2 = dict(m.named_parameters()), dict(tv.named_parameters())
    for k, p in g2.items():
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-6))
        assert err < 1e-3, (k, err)
    err = float((xs.grad.double() - xd.grad).norm() / xd.grad.norm())
    assert err < 1e-3, err


def test_block_composite_equals_torchvision_cnblock_in_float64():
    torch.manual_seed(0)
    C = 24
    ref = TvCNBlock(C, 0.7, 0.0).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(torch.randn_like(p) * 0.2)
    blk = CNBlock(C, 1.0, 0.0).double()
    blk.load_state_dict(ref.state_dict())
    x = torch.randn(3, C, 9, 11, dtype=torch.float64, requires_grad=True)
    xr = x.detach().clone().requires_grad_(True)
    z, zr = blk(x), ref(xr)
    assert torch.allclose(z, zr, atol=1e-12, rtol=1e-12)
    g = torch.randn_like(z)
    z.backward(g)
    zr.backward(g)
    assert torch.allclose(x.grad, xr.grad, atol=1e-12, rtol=1e-10)
    for (k, p), (_, q) in zip(blk.named_parameters(), ref.named_parameters()):
        assert torch.allclose(p.grad, q.grad, atol=1e-12, rtol=1e-10), k
    # stochastic depth: a dropped sample is its input, a kept one is scaled by 1 / (1 - p)
    keep = torch.tensor([0.0, 2.0, 2.0], dtype=torch.float64)
    d = blk.block
    z = ops.convnext_block(x, d[0].weight, d[0].bias, d[2].weight, d[2].bias, 1e-6, d[3].weight, d[3].bias, d[5].weight,
                           d[5].bias, blk.layer_scale, keep)
    base = ops.convnext_block(x, d[0].weight, d[0].bias, d[2].weight, d[2].bias, 1e-6, d[3].weight, d[3].bias,
                              d[5].weight, d[5].bias, blk.layer_scale, None)
    assert torch.equal(z[0], x[0]) and torch.allclose(z[1:] - x[1:], 2 * (base[1:] - x[1:]), atol=1e-12)


def test_layer_norm_composite_equals_layernorm2d_and_layernorm():
    torch.manual_seed(0)
    ref = LayerNorm2d(40, eps=1e-6).double()
    with torch.no_grad():
        ref.weight.add_(torch.randn(40, dtype=torch.float64))
        ref.bias.add_(torch.randn(40, dtype=torch.float64))
    ln = LayerNorm(40, eps=1e-6).double()
    ln.load_state_dict(ref.state_dict())
    x = (torch.randn(2, 40, 5, 3, dtype=torch.float64) * 0.01 + 100.0)       # mean far larger than the spread
    assert torch.allclose(ln(x), ref(x), atol=1e-10, rtol=1e-10)
    x2 = torch.randn(6, 40, dtype=torch.float64)
    assert torch.allclose(ln(x2), F.layer_norm(x2, (40,), ln.weight, ln.bias, 1e-6), atol=1e-12)
    assert list(ln.state_dict()) == list(torch.nn.LayerNorm(40).state_dict())


def test_supports_depthwise7_and_the_existing_predicates():
    assert native.supports_depthwise7(96, (7, 7), 1, 3, 1, 96) and native.supports_depthwise7(8, 7, 1, 3, 1, 8)
    for args in ((96, (7, 7), 2, 3, 1, 96), (96, (7, 7), 1, 2, 1, 96), (100, (7, 7), 1, 3, 1, 100),
                 (96, (7, 7), 1, 3, 2, 96), (96, (5, 5), 1, 2, 1, 96), (96, (7, 7), 1, 3, 1, 48)):
        assert not native.supports_depthwise7(*args), args
    # the 3x3 / 5x5 predicates keep their answers: a 7x7 layer is not a conv_bn_act depthwise layer
    assert not native.supports_depthwise(96, (7, 7), 1, 3, 1, 96) and not native.supports_depthwise5(96, (7, 7), 1, 3, 1, 96)
    assert not native.depthwise_native(96, (7, 7), 1, 3, 1, 96)
    assert native.depthwise_native(96, (3, 3), 2, 1, 1, 96) and native.depthwise_native(96, (5, 5), 1, 2, 1, 96)
    assert all(native.supports_layer_norm(c) for c in (8, 96, 128, 192, 256, 384, 512, 768, 1024, 1536))
    assert not native.supports_layer_norm(8 * 7 * 32 * 2) and not native.supports_layer_norm(100)


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
            cur = re.sub(r"^(void )?ddl::|\(.*\)$", "", cur.replace("(anonymous namespace)::", ""))
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
    dw7 = _ptxas("depthwise7.cu")
    assert sorted(dw7) == ["dwconv7_l1_kernel<false>", "dwconv7_l1_kernel<true>", "dwconv7_tile_kernel<false>",
                           "dwconv7_tile_kernel<true>", "dwconv7_wgrad_kernel"], sorted(dw7)
    bounds = {"tile": 64, "l1": 85, "wgrad": 128}            # __launch_bounds__(256, 4) / (256, 3) / (256, 2)
    for n, (regs, st, ld) in dw7.items():
        assert st == 0 and ld == 0 and regs <= bounds[n.split("_")[1]], (n, regs)
    cx = _ptxas("convnext.cu")
    assert len(cx) == 16, sorted(cx)            # LayerNorm fwd / bwd for V = 1..6, GELU fwd / bwd, layer scale fwd / bwd
    for n, (regs, st, ld) in cx.items():
        v = re.search(r"<(\d+)>", n)
        bound = 255
        if v and "fwd" in n and int(v.group(1)) <= 5 or v and "bwd" in n and int(v.group(1)) <= 3:
            bound = 128                         # two blocks of 256 threads per SM
        assert st == 0 and ld == 0 and regs <= bound, (n, regs, st, ld)
