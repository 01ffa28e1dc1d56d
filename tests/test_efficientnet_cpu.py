"""EfficientNet-B0 to -B7 on CPU: torchvision parity (state_dict, parameter counts, BN settings, dropout, input sizes,
depthwise and squeeze-excitation tables, initialisation, train-mode forward / gradients / running statistics with the
same stochastic-depth draws, eval logits), the SiLU BN, SiLU squeeze-excitation and stochastic-depth composites, and
the compiled SiLU BN / stochastic-depth BN / sigmoid squeeze-excitation kernels (ptxas)."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.ops import SqueezeExcitation, StochasticDepth

from distributeddeeplearning_b200 import _ext, models, ops
from distributeddeeplearning_b200.models.efficientnet import ConvBNAct, MBConv, SqueezeExcitation as SE
from distributeddeeplearning_b200.ops import native

NAMES = [f"efficientnet_b{i}" for i in range(8)]
PARAMS = dict(zip(NAMES, [5_288_548, 7_794_184, 9_109_994, 12_233_232, 19_341_616, 30_389_784, 43_040_704, 66_347_960]))
DROPOUT = dict(zip(NAMES, [0.2, 0.2, 0.3, 0.3, 0.4, 0.4, 0.5, 0.5]))
HEAD = dict(zip(NAMES, [1280, 1280, 1408, 1536, 1792, 2048, 2304, 2560]))
SIZE = dict(zip(NAMES, [224, 240, 288, 300, 380, 456, 528, 600]))
# EfficientNet-B0's depthwise layers as (C, H=W of the input, kernel, stride) and its SE units as (C, C')
DW_B0 = [(32, 112, 3, 1), (96, 112, 3, 2), (144, 56, 3, 1), (144, 56, 5, 2), (240, 28, 5, 1), (240, 28, 3, 2),
         (480, 14, 3, 1), (480, 14, 3, 1), (480, 14, 5, 1), (672, 14, 5, 1), (672, 14, 5, 1), (672, 14, 5, 2),
         (1152, 7, 5, 1), (1152, 7, 5, 1), (1152, 7, 5, 1), (1152, 7, 3, 1)]
SE_B0 = [(32, 8), (96, 4), (144, 6), (144, 6), (240, 10), (240, 10), (480, 20), (480, 20), (480, 20), (672, 28),
         (672, 28), (672, 28), (1152, 48), (1152, 48), (1152, 48), (1152, 48)]


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_params_bn_dropout_and_input_size_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    assert list(m.state_dict()) == list(tv.state_dict())
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in tv.state_dict().items()}
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == PARAMS[name]
    eps, mom = (1e-3, 0.01) if name in NAMES[5:] else (1e-5, 0.1)
    for mod in m.modules():
        if hasattr(mod, "running_var"):
            assert mod.eps == eps and mod.momentum == mom
    assert m.classifier[0].p == tv.classifier[0].p == DROPOUT[name]
    assert m.last_channel == HEAD[name] == tv.classifier[1].in_features
    assert models.input_size(name) == m.input_size == SIZE[name]
    # stochastic depth: 0.2 * block index / blocks, applied only on blocks that keep their shape
    blocks, tvb = [b for b in m.modules() if isinstance(b, MBConv)], [b for b in tv.modules()
                                                                      if type(b).__name__ == "MBConv"]
    assert [(b.use_res_connect, b.sd_prob) for b in blocks] == [(b.use_res_connect, b.stochastic_depth.p) for b in tvb]
    if name == "efficientnet_b0":
        assert len(blocks) == 16 and sum(b.use_res_connect for b in blocks) == 9


def _dw_and_se(m):
    dws, ses, hw = [], [], (m.input_size - 1) // 2 + 1
    for blk in (b for b in m.modules() if isinstance(b, MBConv)):
        for mod in blk.block:
            if isinstance(mod, ConvBNAct) and mod[0].groups > 1:
                c, k, s = mod[0].in_channels, mod[0].kernel_size[0], mod[0].stride
                assert mod[0].groups == c == mod[0].out_channels and mod[0].padding == k // 2
                dws.append((c, hw, k, s))
                hw = (hw - 1) // s + 1
            elif isinstance(mod, SE):
                ses.append((mod.fc1.in_channels, mod.fc1.out_channels))
    return dws, ses


def _tv_dw_and_se(tv, size):
    dws, ses, hw = [], [], (size - 1) // 2 + 1
    for blk in (b for b in tv.modules() if type(b).__name__ == "MBConv"):
        for mod in blk.block:
            if isinstance(mod, SqueezeExcitation):
                ses.append((mod.fc1.in_channels, mod.fc1.out_channels))
            elif mod[0].groups > 1:
                c, k, s = mod[0].in_channels, mod[0].kernel_size[0], mod[0].stride[0]
                dws.append((c, hw, k, s))
                hw = (hw - 1) // s + 1
    return dws, ses


@pytest.mark.parametrize("name", ["efficientnet_b0", "efficientnet_b7"])
def test_depthwise_and_se_layers_are_the_table(name):
    dws, ses = _dw_and_se(models.get_model(name))
    assert (dws, ses) == _tv_dw_and_se(getattr(torchvision.models, name)(), SIZE[name])
    if name == "efficientnet_b0":
        assert dws == DW_B0 and ses == SE_B0
    for c, _, k, s in dws:
        assert native.depthwise_native(c, (k, k), s, k // 2, 1, c), (c, k, s)
    assert any(cs % 8 != 0 for _, cs in ses)          # squeeze widths the hardsigmoid SE node would refuse


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m = models.get_model("efficientnet_b0")
    bn = m.features[2][0].block[0][1]
    assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))
    fw, fb = m.classifier[1].weight.detach(), m.classifier[1].bias.detach()
    r = 1.0 / 1000 ** 0.5
    assert torch.equal(fb, torch.zeros_like(fb))
    assert float(fw.abs().max()) <= r and abs(float(fw.std()) - r / 3 ** 0.5) < 0.05 * r
    se = m.features[6][1].block[2]
    assert isinstance(se, SE)
    for conv in (se.fc1, se.fc2):
        assert torch.equal(conv.bias, torch.zeros_like(conv.bias))
    w = m.features[6][1].block[1][0].weight         # depthwise [1152, 1, 5, 5]: kaiming normal, fan_out = 1152 * 25
    assert tuple(w.shape) == (1152, 1, 5, 5)
    ref = (2.0 / (1152 * 25)) ** 0.5
    assert abs(float(w.detach().std()) - ref) < 0.05 * ref
    assert w.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("name", ["efficientnet_b0", "efficientnet_b1"])
def test_train_forward_backward_equals_torchvision_with_the_same_stochastic_depth(name, monkeypatch):
    torch.manual_seed(3)
    m, tv = models.get_model(name), getattr(torchvision.models, name)()
    m.load_state_dict(tv.state_dict())
    tv = tv.double()          # small batches make BN backward ill-conditioned: compare against float64
    m.train(), tv.train()
    m.classifier[0].p = tv.classifier[0].p = 0.0      # dropout masks come from different generators
    keeps, draw = [], ops.stochastic_depth_keep

    def record(n, p, device):
        keeps.append(draw(n, p, device))
        return keeps[-1]

    monkeypatch.setattr(ops, "stochastic_depth_keep", record)
    replay = []
    monkeypatch.setattr(StochasticDepth, "forward",
                        lambda self, x: x if self.p == 0.0 else x * replay.pop(0).view(-1, 1, 1, 1).to(x.dtype))
    x = torch.randn(4, 3, 96, 96)
    y = torch.tensor([1, 7, 3, 9])
    o1 = m(x)
    replay[:] = keeps
    o2 = tv(x.double())
    assert not replay and len(keeps) == sum(b.use_res_connect and b.sd_prob > 0 for b in m.modules()
                                            if isinstance(b, MBConv))
    assert sum(int((k == 0).sum()) for k in keeps) > 0          # some sample was dropped by some block
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
    x = torch.randn(2, 3, 64, 48)
    with torch.no_grad():
        assert torch.allclose(m(x), tv(x), atol=1e-4, rtol=1e-4)


@pytest.mark.parametrize("c,cs", [(32, 8), (96, 4), (144, 6), (240, 10), (1152, 48), (3840, 160)])
def test_silu_squeeze_excite_equals_torchvision(c, cs):
    torch.manual_seed(0)
    ref = SqueezeExcitation(c, cs, activation=torch.nn.SiLU).double()
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(torch.randn_like(p) * 0.5)
    w1, b1, w2, b2 = (p.detach().clone().requires_grad_(True) for p in
                      (ref.fc1.weight, ref.fc1.bias, ref.fc2.weight, ref.fc2.bias))
    x = (torch.randn(3, c, 5, 6, dtype=torch.float64) * 3).requires_grad_(True)
    xr = x.detach().clone().requires_grad_(True)
    y = ops.squeeze_excite(x, w1, b1, w2, b2, gate="sigmoid", act="silu")
    yr = ref(xr)
    assert torch.allclose(y, yr, atol=1e-12, rtol=1e-12)
    g = torch.randn_like(y)
    y.backward(g)
    yr.backward(g)
    assert torch.allclose(x.grad, xr.grad, atol=1e-12, rtol=1e-10)
    for got, p in zip((w1, b1, w2, b2), (ref.fc1.weight, ref.fc1.bias, ref.fc2.weight, ref.fc2.bias)):
        assert torch.allclose(got.grad, p.grad, atol=1e-12, rtol=1e-10)
    with pytest.raises(ValueError):
        ops.squeeze_excite(x, w1, b1, w2, b2, gate="sigmoid", act="relu")


def test_silu_bn_composite_equals_silu_of_batch_norm():
    torch.manual_seed(0)
    x = torch.randn(3, 16, 9, 7) * 4
    w = torch.randn(16, 16, 3, 3) * 0.5
    g, b = torch.rand(16) + 0.5, torch.randn(16)
    for training in (True, False):
        rm1, rv1 = torch.randn(16) * 0.1, torch.rand(16) + 0.5
        rm2, rv2 = rm1.clone(), rv1.clone()
        z = ops.conv_bn_act(x, w, g, b, rm1, rv1, 1, 1, training=training, silu=True)
        v = F.batch_norm(F.conv2d(x, w, None, 1, 1), rm2, rv2, g, b, training)
        assert torch.allclose(z, F.silu(v), atol=1e-5, rtol=1e-5)
        assert 0.2 < float((v > 0).float().mean()) < 0.8                   # straddles 0
        assert torch.allclose(rm1, rm2) and torch.allclose(rv1, rv2)
    wd = torch.randn(16, 1, 5, 5)                                            # depthwise 5x5 composite with SiLU
    z = ops.conv_bn_act(x, wd, g, b, torch.zeros(16), torch.ones(16), 2, 2, groups=16, silu=True)
    ref = F.silu(F.batch_norm(F.conv2d(x, wd, None, 2, 2, 1, 16), torch.zeros(16), torch.ones(16), g, b, True))
    assert torch.allclose(z, ref, atol=1e-5, rtol=1e-5)
    rm, rv = torch.zeros(16), torch.ones(16)
    for kw in ({"residual": x}, {"relu6": True}, {"hardswish": True}):
        with pytest.raises(ValueError):
            ops.conv_bn_act(x, w, g, b, rm, rv, 1, 1, silu=True, **kw)


def test_stochastic_depth_composite_scales_the_bn_output_per_sample():
    torch.manual_seed(0)
    x = torch.randn(4, 16, 6, 6)
    r = torch.randn(4, 24, 6, 6)
    w = torch.randn(24, 16, 1, 1) * 0.3
    g, b = torch.rand(24) + 0.5, torch.randn(24)
    keep = torch.tensor([1.25, 0.0, 1.25, 1.25])
    rm1, rv1, rm2, rv2 = torch.zeros(24), torch.ones(24), torch.zeros(24), torch.ones(24)
    xs, rs = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    z = ops.conv_bn_act(xs, w, g, b, rm1, rv1, relu=False, residual=rs, sample_scale=keep)
    xr, rr = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    zr = F.batch_norm(F.conv2d(xr, w), rm2, rv2, g, b, True) * keep.view(-1, 1, 1, 1) + rr
    assert torch.allclose(z, zr, atol=1e-5, rtol=1e-5)
    assert torch.equal(z[1], r[1])                                           # a dropped sample is its shortcut
    assert torch.allclose(rm1, rm2) and torch.allclose(rv1, rv2)             # statistics over every sample
    dz = torch.randn_like(z)
    z.backward(dz)
    zr.backward(dz)
    assert torch.allclose(xs.grad, xr.grad, atol=1e-5, rtol=1e-5) and torch.equal(rs.grad, dz)
    rm, rv = torch.zeros(24), torch.ones(24)
    for kw in ({"residual": None}, {"relu": True}, {"training": False}):
        with pytest.raises(ValueError):
            ops.conv_bn_act(x, w, g, b, rm, rv, **{"relu": False, "residual": r, **kw}, sample_scale=keep)
    k = ops.stochastic_depth_keep(10_000, 0.2, "cpu")
    assert set(k.unique().tolist()) == {0.0, 1.25} and abs(float((k > 0).float().mean()) - 0.8) < 0.02


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
            cur = re.sub(r"^void ddl::|\(.*\)$", "", cur.replace("(anonymous namespace)::", ""))
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
    bn = _ptxas("bn_act.cu")
    new = [n for n in bn if n.startswith(("bn_silu_fwd_kernel", "bn_sd_fwd_kernel")) or re.search(r"<[78][,>]", n)]
    # SiLU fwd train / eval x flat / chunked, stochastic-depth fwd flat / chunked; reduce and apply (flat / chunked) of
    # masks 7 (SiLU) and 8 (stochastic depth)
    assert len(new) == 12, sorted(new)
    for n in new:
        assert bn[n][1:] == [0, 0] and bn[n][0] <= 64, (n, bn[n])          # __launch_bounds__(256, 4)
    se = _ptxas("squeeze_excite_sigmoid.cu")
    assert len(se) == 5, sorted(se)
    misc = {n: v for n, v in _ptxas("misc_ops.cu").items() if "silu_rows" in n or "stochastic_depth" in n}
    assert len(misc) == 3, sorted(misc)
    for name, (regs, st, ld) in list(se.items()) + list(misc.items()):
        assert st == 0 and ld == 0 and regs <= 255, (name, regs, st, ld)
