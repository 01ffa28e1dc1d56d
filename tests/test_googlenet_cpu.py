"""GoogLeNet on CPU: torchvision parity (state_dict with and without the auxiliary heads, parameter counts,
initialisation, eval logits and train-mode outputs and gradients in float64), the Inception module composite against
torchvision's ``Inception`` at every module shape, the adaptive average pool composite, the shared auxiliary-loss rule
of the trainers, and the compiled kernels of csrc/ops/inception.cu (ptxas)."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F
import torchvision
from torchvision.models.googlenet import Inception as TvInception

from distributeddeeplearning_b200 import _ext, models, ops
from distributeddeeplearning_b200.ops.googlenet import inception_module_composite

# (cin, c1, c2r, c2, c3r, c3, c4, spatial size) of the nine modules
MODULES = [(192, 64, 96, 128, 16, 32, 32, 28), (256, 128, 128, 192, 32, 96, 64, 28), (480, 192, 96, 208, 16, 48, 64, 14),
           (512, 160, 112, 224, 24, 64, 64, 14), (512, 128, 128, 256, 24, 64, 64, 14),
           (512, 112, 144, 288, 32, 64, 64, 14), (528, 256, 160, 320, 32, 128, 128, 14),
           (832, 256, 160, 320, 32, 128, 128, 7), (832, 384, 192, 384, 48, 128, 128, 7)]


def _randomize(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in model.modules():
            if hasattr(mod, "running_var") and mod.running_var is not None:
                c = mod.running_var.numel()
                mod.weight.copy_(torch.rand(c, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(c, generator=g) * 0.3)
                mod.running_mean.copy_(torch.randn(c, generator=g) * 0.2)
                mod.running_var.copy_(torch.rand(c, generator=g) + 0.5)


def _tv(**kw):
    return torchvision.models.googlenet(init_weights=True, **kw)


@pytest.mark.parametrize("aux,count", [(True, 13_004_888), (False, 6_624_904)])
def test_state_dict_and_parameter_count_match_torchvision(aux, count):
    m = models.get_model("googlenet", aux_logits=aux)
    tv = _tv(aux_logits=aux)
    sd, tsd = m.state_dict(), tv.state_dict()
    assert list(sd) == list(tsd)
    assert [(tuple(v.shape), v.dtype) for v in sd.values()] == [(tuple(v.shape), v.dtype) for v in tsd.values()]
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == count
    assert ("aux1.fc2.weight" in sd) == aux and "inception4e.branch4.1.conv.weight" in sd
    assert models.input_size("googlenet") == models.input_size(m) == 224
    # checkpoints load strictly in both directions
    tv.load_state_dict(m.state_dict(), strict=True)
    m.load_state_dict(tv.state_dict(), strict=True)


def test_builder_arguments():
    m = models.get_model("googlenet", num_classes=10, aux_logits=True, transform_input=True, init_weights=False,
                         dropout=0.3, dropout_aux=0.6)
    assert m.fc.out_features == 10 and m.aux1.fc2.out_features == 10 and m.p == 0.3 and m.aux2.p == 0.6
    assert m.transform_input and m.aux_loss_weight == 0.3
    with pytest.raises(ValueError):
        models.get_model("googlenet", blocks=[object, object, object])
    with pytest.raises(ValueError):
        models.get_model("googlenet", pretrained=True)


def test_initialisation_matches_torchvision():
    torch.manual_seed(0)
    m = models.get_model("googlenet")
    for name, p in m.named_parameters():
        if p.dim() >= 2:               # trunc_normal_(std=0.01, a=-2, b=2): the bounds are 200 std away
            assert abs(p.std().item() - 0.01) < 0.1 * 0.01 + 2e-3 * (p.numel() < 2000), name
            assert abs(p.mean().item()) < 3e-3, name
        elif name.endswith("bn.weight"):
            assert torch.equal(p, torch.ones_like(p)), name
        elif name.endswith("bn.bias"):
            assert torch.equal(p, torch.zeros_like(p)), name
    for b in m.modules():
        if hasattr(b, "running_var"):
            assert b.eps == 0.001 and b.momentum == 0.1


def test_eval_logits_match_torchvision_float64():
    torch.manual_seed(1)
    tv = _tv(transform_input=True)
    _randomize(tv, 7)
    m = models.get_model("googlenet", transform_input=True)
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.double().eval()
    x = torch.randn(2, 3, 224, 224)
    with torch.no_grad():
        got, ref = m(x).double(), tv(x.double())
    assert got.shape == (2, 1000)
    assert float((got - ref).abs().max()) <= 1e-4 * float(ref.abs().max()) + 1e-9


def test_train_outputs_and_gradients_match_torchvision_float64():
    torch.manual_seed(2)
    tv = _tv()
    _randomize(tv, 3)
    m = models.get_model("googlenet", dropout=0.0, dropout_aux=0.0)
    m.load_state_dict(tv.state_dict())
    tv.dropout.p = 0.0
    tv.aux1.dropout.p = tv.aux2.dropout.p = 0.0
    m.train(), tv.double().train()          # small batches make BN backward ill-conditioned: compare against float64
    x = torch.randn(8, 3, 128, 128)
    y = torch.tensor([1, 5, 9, 3, 0, 7, 2, 8])
    o1, o2 = m(x), tv(x.double())
    assert type(o1).__name__ == "GoogLeNetOutputs" and o1._fields == ("logits", "aux_logits2", "aux_logits1")
    for a, b in zip(o1, o2):
        assert torch.allclose(a.double(), b, atol=5e-4, rtol=1e-3)
    l1 = ops.aux_classification_loss(o1, y, 1000, m.aux_loss_weight)
    l2 = F.cross_entropy(o2[0], y) + 0.3 * (F.cross_entropy(o2[1], y) + F.cross_entropy(o2[2], y))
    assert torch.allclose(l1.double(), l2, rtol=1e-5)
    l1.backward(), l2.backward()
    g1 = dict(m.named_parameters())
    for k, p in tv.named_parameters():
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-4))
        assert err < 5e-2, (k, err)
    tb = dict(tv.named_buffers())
    for k, b in m.named_buffers():
        if "running" in k:
            assert torch.allclose(b.double(), tb[k], atol=1e-5, rtol=1e-4), k


def _layers(tv):
    def bn(b):
        return (b.weight, b.bias, b.running_mean.clone(), b.running_var.clone(), b.eps, b.momentum)

    convs = (tv.branch1, tv.branch2[0], tv.branch2[1], tv.branch3[0], tv.branch3[1], tv.branch4[1])
    return [(c.conv.weight, bn(c.bn)) for c in convs], convs


@pytest.mark.parametrize("shape", MODULES, ids=[f"{s[0]}-{s[1]}" for s in MODULES])
@pytest.mark.parametrize("training", [True, False])
def test_inception_composite_matches_torchvision(shape, training):
    cin, c1, c2r, c2, c3r, c3, c4, hw = shape
    torch.manual_seed(cin + c1)
    tv = TvInception(cin, c1, c2r, c2, c3r, c3, c4).double()
    _randomize(tv, c2)
    tv.train(training)
    layers, convs = _layers(tv)
    x = torch.randn(2, cin, hw, hw, dtype=torch.float64, requires_grad=True)
    ref = tv(x)
    xc = x.detach().clone().requires_grad_(True)
    got = inception_module_composite(xc, layers, training)
    assert got.shape == (2, c1 + c2 + c3 + c4, hw, hw)
    assert torch.allclose(got, ref, rtol=1e-10, atol=1e-10)
    for (_, ours), c in zip(layers, convs):
        assert torch.allclose(ours[2], c.bn.running_mean, rtol=1e-12, atol=1e-14)
        assert torch.allclose(ours[3], c.bn.running_var, rtol=1e-12, atol=1e-14)
    ref.backward(torch.ones_like(ref))
    got.backward(torch.ones_like(got))
    assert torch.allclose(xc.grad, x.grad, rtol=1e-9, atol=1e-10)


def test_inception_module_runs_the_composite_on_cpu():
    torch.manual_seed(4)
    from distributeddeeplearning_b200.models.googlenet import Inception

    ours, tv = Inception(480, 192, 96, 208, 16, 48, 64), TvInception(480, 192, 96, 208, 16, 48, 64)
    _randomize(tv, 5)
    ours.load_state_dict(tv.state_dict())
    x = torch.randn(2, 480, 14, 14)
    assert torch.allclose(ours(x), tv(x), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("hw,out", [((14, 14), (4, 4)), ((7, 9), (3, 4)), ((5, 5), (5, 5)), ((13, 11), (1, 1)),
                                    ((17, 14), (6, 4))])
def test_adaptive_avg_pool_composite_matches_torch(hw, out):
    x = torch.randn(2, 16, *hw, dtype=torch.float64)
    assert torch.equal(ops.adaptive_avg_pool2d(x, out), F.adaptive_avg_pool2d(x, out))
    assert torch.equal(ops.flatten_nchw(x), torch.flatten(x, 1))


def test_aux_loss_rule():
    torch.manual_seed(5)
    y = torch.tensor([0, 3, 2])
    main, a1, a2 = (torch.randn(3, 10, dtype=torch.float64) for _ in range(3))
    assert models.get_model("inception_v3", aux_logits=False).aux_loss_weight == 0.4
    xent = ops.softmax_cross_entropy
    # Inception-v3's (logits, aux): exactly the trainers' former main + 0.4 aux
    got = ops.aux_classification_loss((main, a1), y, 10, 0.4)
    assert torch.equal(got, xent(main, y, 10) + 0.4 * xent(a1, y, 10))
    # GoogLeNet's (logits, aux2, aux1): main + 0.3 (aux1 + aux2)
    got = ops.aux_classification_loss((main, a2, a1), y, 10, 0.3)
    ref = F.cross_entropy(main, y) + 0.3 * (F.cross_entropy(a1, y) + F.cross_entropy(a2, y))
    assert torch.allclose(got.double(), ref, rtol=1e-6)
    assert torch.equal(ops.aux_classification_loss(main, y, 10, None), xent(main, y, 10))
    with pytest.raises(ValueError):
        ops.aux_classification_loss((main, a1), y, 10, None)


def test_trainers_share_the_aux_loss_rule():
    root = os.path.join(os.path.dirname(_ext.__file__), "workloads")
    for f in ("benchmark.py", "imagenet.py", "hvd_imagenet.py"):
        src = open(os.path.join(root, f)).read()
        assert "aux_classification_loss" in src and "0.4" not in src, f


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
def test_inception_kernels_compile_without_spills():
    k = _ptxas("inception.cu")
    assert sorted(k) == sorted(["bn_seg_fwd_kernel<true>", "bn_seg_fwd_kernel<false>", "bn_seg_bwd_reduce_kernel",
                                "bn_seg_bwd_apply_kernel", "adaptive_avgpool_fwd_kernel", "adaptive_avgpool_bwd_kernel",
                                "transpose_rows_kernel"]), sorted(k)
    for name, (regs, st, ld) in k.items():
        assert st == 0 and ld == 0, (name, regs, st, ld)
        if name.startswith("bn_seg"):          # __launch_bounds__(256, 4): 4 CTAs / SM, like the BN kernels
            assert regs <= 64, (name, regs)


def test_new_kernels_are_counted():
    for name, n in (("bn_seg_fwd", 1), ("bn_seg_bwd", 2), ("adaptive_avgpool_fwd", 1), ("adaptive_avgpool_bwd", 1),
                    ("transpose_rows", 1)):
        assert _ext.KERNEL_LAUNCHES[name] == n
    src = open(os.path.join(os.path.dirname(_ext.__file__), "csrc", "ops", "inception.cu")).read()
    assert "<<<" not in src and src.count("launch_pdl(") >= 6
