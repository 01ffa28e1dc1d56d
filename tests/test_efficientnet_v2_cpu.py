"""EfficientNetV2-S, -M and -L on CPU: torchvision parity (state_dict, parameter counts, block counts, BN settings,
dropout, stochastic-depth probabilities, input sizes, initialisation, eval logits, and train-mode logits / gradients /
running statistics with the same stochastic-depth draws), the Fused-MBConv conv shapes, the composites of the
Fused-MBConv node in both forms, the refusals the new BN mode leaves in place, and the compiled SiLU-before-residual BN
kernels (ptxas)."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.ops import StochasticDepth

from distributeddeeplearning_b200 import _ext, models, ops
from distributeddeeplearning_b200.models.efficientnet import MBConv
from distributeddeeplearning_b200.models.efficientnet_v2 import FusedMBConv
from distributeddeeplearning_b200.ops import native
from distributeddeeplearning_b200.ops.efficientnet_v2 import fused_mbconv_composite

NAMES = ["efficientnet_v2_s", "efficientnet_v2_m", "efficientnet_v2_l"]
# name: (parameters, state_dict entries, residual Fused-MBConv blocks, Fused-MBConv blocks, MBConv blocks, dropout, crop)
TABLE = {"efficientnet_v2_s": (21_458_488, 782, 8, 10, 30, 0.2, 384),
         "efficientnet_v2_m": (54_139_356, 1_120, 11, 13, 44, 0.3, 480),
         "efficientnet_v2_l": (118_515_272, 1_548, 16, 18, 61, 0.4, 480)}
# the Fused-MBConv convolutions (cin, cout, kernel, stride) of each model
FUSED_S = {(24, 24, 3, 1), (24, 96, 3, 2), (48, 192, 3, 1), (48, 192, 3, 2), (64, 256, 3, 1), (96, 48, 1, 1),
           (192, 48, 1, 1), (192, 64, 1, 1), (256, 64, 1, 1)}
FUSED = {"efficientnet_v2_s": FUSED_S,
         "efficientnet_v2_m": (FUSED_S - {(64, 256, 3, 1), (192, 64, 1, 1), (256, 64, 1, 1)})
         | {(80, 320, 3, 1), (192, 80, 1, 1), (320, 80, 1, 1)},
         "efficientnet_v2_l": {(32, 32, 3, 1), (32, 128, 3, 2), (64, 256, 3, 1), (64, 256, 3, 2), (96, 384, 3, 1),
                               (128, 64, 1, 1), (256, 64, 1, 1), (256, 96, 1, 1), (384, 96, 1, 1)}}


def _blocks(m, kind):
    return [b for b in m.modules() if type(b).__name__ == kind]


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_and_table_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    sd, tsd = m.state_dict(), tv.state_dict()
    assert list(sd) == list(tsd)
    assert [(tuple(v.shape), v.dtype) for v in sd.values()] == [(tuple(v.shape), v.dtype) for v in tsd.values()]
    params, entries, res_fused, fused, mb, dropout, crop = TABLE[name]
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == params
    assert len(sd) == entries
    fb, tfb = _blocks(m, "FusedMBConv"), _blocks(tv, "FusedMBConv")
    assert len(fb) == len(tfb) == fused and sum(b.use_res_connect for b in fb) == res_fused
    assert len(_blocks(m, "MBConv")) == len(_blocks(tv, "MBConv")) == mb
    for mod in m.modules():
        if hasattr(mod, "running_var"):
            assert mod.eps == 1e-3 and mod.momentum == 0.1
    assert m.classifier[0].p == tv.classifier[0].p == dropout
    assert m.last_channel == tv.classifier[1].in_features == 1280
    assert models.input_size(name) == models.input_size(m) == crop
    # stochastic depth: 0.2 * block index / blocks over both block kinds, so the first block has p = 0
    ours = [b for b in m.modules() if isinstance(b, (FusedMBConv, MBConv))]
    theirs = [b for b in tv.modules() if type(b).__name__ in ("FusedMBConv", "MBConv")]
    assert [(type(b).__name__, b.use_res_connect, b.sd_prob) for b in ours] == \
        [(type(b).__name__, b.use_res_connect, b.stochastic_depth.p) for b in theirs]
    assert ours[0].sd_prob == 0.0 and ours[0].use_res_connect
    assert all(abs(b.sd_prob - 0.2 * i / len(ours)) < 1e-12 for i, b in enumerate(ours))


@pytest.mark.parametrize("name", NAMES)
def test_fused_conv_shapes_are_the_table_and_native(name):
    m = models.get_model(name)
    shapes = {(mod[0].in_channels, mod[0].out_channels, mod[0].kernel_size[0], mod[0].stride)
              for b in _blocks(m, "FusedMBConv") for mod in b.block}
    assert shapes == FUSED[name]
    for cin, cout, _, _ in shapes:
        assert native.supports_conv(cin, cout) and native.bn_supported(cout)


def test_builder_arguments_are_torchvisions():
    m = models.get_model("efficientnet_v2_s", num_classes=10, dropout=0.5, stochastic_depth_prob=0.4)
    tv = torchvision.models.efficientnet_v2_s(num_classes=10, dropout=0.5, stochastic_depth_prob=0.4)
    assert m.classifier[1].out_features == 10 and m.classifier[0].p == 0.5
    assert [b.sd_prob for b in m.modules() if isinstance(b, (FusedMBConv, MBConv))] == \
        [b.stochastic_depth.p for b in tv.modules() if type(b).__name__ in ("FusedMBConv", "MBConv")]
    for kw in ({"width_mult": 1.0}, {"norm_layer": None}, {"last_channel": 1280}):
        with pytest.raises(ValueError):
            models.get_model("efficientnet_v2_m", **kw)


def test_initialisation_follows_torchvision():
    torch.manual_seed(0)
    m = models.get_model("efficientnet_v2_s")
    bn = m.features[1][0].block[0][1]
    assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))
    fw, fb = m.classifier[1].weight.detach(), m.classifier[1].bias.detach()
    r = 1.0 / 1000 ** 0.5
    assert torch.equal(fb, torch.zeros_like(fb))
    assert float(fw.abs().max()) <= r and abs(float(fw.std()) - r / 3 ** 0.5) < 0.05 * r
    w = m.features[3][1].block[0][0].weight          # Fused expand conv [256, 64, 3, 3]: kaiming normal, fan_out
    assert tuple(w.shape) == (256, 64, 3, 3) and w.is_contiguous(memory_format=torch.channels_last)
    ref = (2.0 / (256 * 9)) ** 0.5
    assert abs(float(w.detach().std()) - ref) < 0.05 * ref
    se = m.features[4][0].block[2]
    for conv in (se.fc1, se.fc2):
        assert torch.equal(conv.bias, torch.zeros_like(conv.bias))


@pytest.mark.parametrize("name", NAMES)
def test_eval_equals_torchvision(name):
    torch.manual_seed(0)
    m, tv = models.get_model(name, num_classes=10), getattr(torchvision.models, name)(num_classes=10)
    m.load_state_dict(tv.state_dict())
    with torch.no_grad():                            # non-trivial BN statistics, so that eval differs from train
        for mod in tv.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.1)
                mod.running_var.uniform_(0.5, 1.5)
                mod.weight.uniform_(0.5, 1.5)
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.eval()
    tv = tv.double()
    x = torch.randn(2, 3, 64, 48)
    with torch.no_grad():
        o, r = m(x).double(), tv(x.double())
    assert float((o - r).abs().max()) <= 1e-4 * float(r.abs().max()) + 1e-9


def test_train_forward_backward_equals_torchvision_with_the_same_stochastic_depth(monkeypatch):
    torch.manual_seed(3)
    m, tv = models.get_model("efficientnet_v2_s"), torchvision.models.efficientnet_v2_s()
    m.load_state_dict(tv.state_dict())
    tv = tv.double()          # small batches make BN backward ill-conditioned: compare against float64
    m.train(), tv.train()
    m.classifier[0].p = tv.classifier[0].p = 0.0      # dropout masks come from different generators
    for mod in list(m.modules()) + list(tv.modules()):
        if isinstance(mod, (FusedMBConv, MBConv)):
            mod.sd_prob = 0.5 if mod.sd_prob > 0 else 0.0          # drop often enough to hit the Fused blocks
        elif isinstance(mod, StochasticDepth):
            mod.p = 0.5 if mod.p > 0 else 0.0
    keeps, draw = [], ops.stochastic_depth_keep

    def record(n, p, device):
        keeps.append(draw(n, p, device))
        return keeps[-1]

    monkeypatch.setattr(ops, "stochastic_depth_keep", record)
    replay = []
    monkeypatch.setattr(StochasticDepth, "forward",
                        lambda self, x: x if self.p == 0.0 else x * replay.pop(0).view(-1, 1, 1, 1).to(x.dtype))
    x = torch.randn(4, 3, 64, 64)
    y = torch.tensor([1, 7, 3, 9])
    o1 = m(x)
    replay[:] = keeps
    o2 = tv(x.double())
    blocks = [b for b in m.modules() if isinstance(b, (FusedMBConv, MBConv))]
    assert not replay and len(keeps) == sum(b.use_res_connect and b.sd_prob > 0 for b in blocks)
    fused_draws = sum(b.use_res_connect and b.sd_prob > 0 for b in blocks if isinstance(b, FusedMBConv))
    assert fused_draws == 7 and sum(int((k == 0).sum()) for k in keeps[:fused_draws]) > 0
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


def _bn_params(c, dtype=torch.float64):
    return (torch.rand(c, dtype=dtype) + 0.5, torch.randn(c, dtype=dtype), torch.randn(c, dtype=dtype) * 0.1,
            torch.rand(c, dtype=dtype) + 0.5)


@pytest.mark.parametrize("expand", [1, 4])
@pytest.mark.parametrize("keep,training", [(None, True), ("zeros", True), (None, False)])
def test_fused_mbconv_composite_equals_f_ops(expand, keep, training):
    """Both node forms' composite against F ops in float64 (stochastic depth in training only): output, running
    statistics, a dropped sample equal to its shortcut, and the residual's gradient equal to dz (the input gradient minus
    the branch's is dz)."""
    torch.manual_seed(0)
    c, e = 16, 16 * expand
    x = torch.randn(3, c, 7, 6, dtype=torch.float64) * 2
    w1 = torch.randn(e, c, 3, 3, dtype=torch.float64) * (c * 9) ** -0.5
    g1, b1, rm1, rv1 = _bn_params(e)
    w2 = torch.randn(c, e, 1, 1, dtype=torch.float64) * e ** -0.5 if expand > 1 else None
    g2, b2, rm2, rv2 = _bn_params(c) if expand > 1 else (None,) * 4
    k = torch.tensor([2.0, 0.0, 2.0], dtype=torch.float64) if keep else None
    stats = [t.clone() for t in (rm1, rv1) + ((rm2, rv2) if expand > 1 else ())]
    two = () if expand == 1 else (w2, g2, b2, rm2, rv2, 1e-3, 0.1)
    xs = x.clone().requires_grad_(True)
    z = fused_mbconv_composite(xs, w1, g1, b1, rm1, rv1, 1e-3, 0.1, training, *two, keep=k)
    h = F.silu(F.batch_norm(F.conv2d(x, w1, None, 1, 1), stats[0], stats[1], g1, b1, training, 0.1, 1e-3))
    if expand > 1:
        h = F.batch_norm(F.conv2d(h, w2), stats[2], stats[3], g2, b2, training, 0.1, 1e-3)
    ref = (h * k.view(-1, 1, 1, 1) if k is not None else h) + x
    assert torch.allclose(z, ref, atol=1e-12, rtol=1e-12)
    assert all(torch.allclose(a, b, atol=1e-14) for a, b in zip((rm1, rv1) + ((rm2, rv2) if expand > 1 else ()), stats))
    if k is not None:
        assert torch.equal(z[1], x[1])
    dz = torch.randn_like(z)
    z.backward(dz)
    xb = x.clone().requires_grad_(True)
    branch = fused_mbconv_composite(xb, w1, g1, b1, rm1.clone(), rv1.clone(), 1e-3, 0.1, training,
                                    *((w2, g2, b2, rm2.clone(), rv2.clone(), 1e-3, 0.1) if expand > 1 else ()),
                                    keep=k) - xb
    branch.backward(dz)
    assert torch.allclose(xs.grad - xb.grad, dz, atol=1e-12)


def test_fused_mbconv_on_cpu_takes_the_composite_and_block_zero_draws_nothing():
    torch.manual_seed(0)
    m = models.get_model("efficientnet_v2_s").train()
    blk = m.features[1][0]
    assert blk.sd_prob == 0.0 and blk.use_res_connect and len(blk.block) == 1
    x = torch.randn(2, 24, 8, 8)
    assert not ops.fused_mbconv_supported(x, blk.block[0][0], blk.block[0][1])
    c, bn = blk.block[0]
    ref = F.silu(F.batch_norm(F.conv2d(x, c.weight, None, 1, 1), bn.running_mean.clone(), bn.running_var.clone(),
                              bn.weight, bn.bias, True, 0.1, 1e-3)) + x
    assert torch.allclose(blk(x), ref, atol=1e-5, rtol=1e-5)


def test_existing_refusals_still_raise():
    torch.manual_seed(0)
    x = torch.randn(2, 16, 5, 5)
    w = torch.randn(16, 16, 3, 3)
    g, b, rm, rv = torch.rand(16) + 0.5, torch.randn(16), torch.zeros(16), torch.ones(16)
    keep = torch.tensor([1.25, 0.0])
    with pytest.raises(ValueError):            # SiLU with a residual
        ops.conv_bn_act(x, w, g, b, rm, rv, 1, 1, silu=True, residual=x)
    for kw in ({"silu": True}, {"relu": True}, {"gelu": True}):      # a per-sample scale with an activation
        with pytest.raises(ValueError):
            ops.conv_bn_act(x, w, g, b, rm, rv, 1, 1, **{"relu": False, **kw}, residual=x, sample_scale=keep)


def _ptxas(src):
    """{demangled kernel name: [registers, spill store bytes, spill load bytes, stack bytes]} of one .cu file."""
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
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = [0, int(m.group(2)), int(m.group(3)), int(m.group(1))]
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            out[cur][0] = int(m.group(1))
    return out


@pytest.mark.skipif(not (shutil.which("c++filt") and os.path.isfile(os.path.join(_ext.CUDA_HOME, "bin", "nvcc"))),
                    reason="needs nvcc and c++filt")
def test_new_kernels_compile_without_spills_and_fit_their_launch_bounds():
    bn = _ptxas("bn_act.cu")
    new = sorted(n for n in bn if n.startswith("bn_silu_res_fwd_kernel") or re.search(r"<10[,>]", n))
    # forward train / eval x flat / chunked; reduce and apply (flat / chunked) of mask 10
    assert new == ["bn_act_bwd_apply_kernel<10, false, false>", "bn_act_bwd_apply_kernel<10, true, false>",
                   "bn_act_bwd_reduce_kernel<10>", "bn_silu_res_fwd_kernel<false, false>",
                   "bn_silu_res_fwd_kernel<false, true>", "bn_silu_res_fwd_kernel<true, false>",
                   "bn_silu_res_fwd_kernel<true, true>"], new
    for n in new:
        assert bn[n][1:] == [0, 0, 0] and bn[n][0] <= 64, (n, bn[n])          # __launch_bounds__(256, 4)
